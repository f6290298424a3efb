"""Fused scene assembly (SURVEY.md section 8 f2) - additive API, the reference API is untouched.

``assemble_scene(groups, ...)`` replaces the per-view PyTorch glue of DreamScene's ``scene_render``
(/root/reference/scene_gaussian.py:753-857 with the activations of gs_renderer.py:464-488):

    means3D   = cat([g.get_xyz ...])                       # _xyz
    opacity   = cat([sigmoid(g._opacity) ...])
    scales    = cat([exp(g._scaling) ...])
    rotations = cat([normalize(g._rotation) ...])
    shs       = cat([cat((g._features_dc, g._features_rest), dim=1) ...])
    shs       = shs + randn_like(shs) * (0.2**0.5 * shs)                         # scene_gaussian.py:848-851
    scales    = clamp(scales + randn_like(scales) * (0.2**0.5 * scales / 4), 0)   # :853-856

with ONE kernel forward and ONE kernel backward (dreamscene_b200/csrc/assemble.cu): every raw leaf is
read once, the five packed rasterizer inputs are written once, and the backward writes the leaf
gradients directly (no torch.cat / split / per-op autograd nodes).

Each group is a dict (or any object with these attributes) of the raw leaf tensors
``_xyz [n,3], _opacity [n,1], _scaling [n,3], _rotation [n,4], _features_dc [n,1,3],
_features_rest [n,M-1,3]`` - exactly the attributes of the reference's GaussianModel.

Noise modes
  noise="torch"  : the standard-normal draws come from torch.randn in the reference's order
                   (shs first, then scales): same RNG stream, same values as the reference code.
  noise="fused"  : counter-based Philox evaluated inside the kernels (no noise tensor is written or
                   read; statistically equivalent, not stream-compatible with torch).
  shs_aug / scale_aug = False switch the respective augmentation off (the reference draws
  ``random.random() < ratio`` on the host for that decision: pass its outcome).

``render_scene(groups, settings_list, ...)`` goes one step further: the B views of a training step rendered straight
from the raw groups, with the activations and the Philox augmentation inside the projection kernels (no augmented copy
of shs / scales and no per-view gradient of them is ever written); the rasterizer inputs are bit for bit those of
assemble_scene(noise="fused", views=B) + multiview.rasterize_views for the same seed.
"""
from __future__ import annotations

import ctypes as C
from typing import Sequence

import torch

from . import _lib

_FIELDS = ("_xyz", "_opacity", "_scaling", "_rotation", "_features_dc", "_features_rest")
NOISE_COEF = 0.2 ** 0.5      # scene_gaussian.py:849,854


def _get(group, name):
    return group[name] if isinstance(group, dict) else getattr(group, name)


def _group_table(raw: Sequence[Sequence[torch.Tensor]]):
    arr = (_lib.Group * len(raw))()
    for k, ts in enumerate(raw):
        for name, t in zip(("xyz", "opacity", "scaling", "rotation", "f_dc", "f_rest"), ts):
            setattr(arr[k], name, t.data_ptr() if t.numel() else None)
        arr[k].n = int(ts[0].shape[0])
    return arr


class _Assemble(torch.autograd.Function):
    @staticmethod
    def forward(ctx, num_groups, M, B, c_shs, c_scale, z_shs, z_scales, seed, *flat):
        raw = [[_lib.prepare(t.detach()) for t in flat[6 * k:6 * k + 6]] for k in range(num_groups)]
        dev = raw[0][0].device
        P = sum(int(ts[0].shape[0]) for ts in raw)
        out = [torch.empty(P, 3, device=dev), torch.empty(P, 1, device=dev), torch.empty(B, P, 3, device=dev),
               torch.empty(P, 4, device=dev), torch.empty(B, P, M, 3, device=dev)]
        lib, ptr = _lib.load(), _lib.ptr
        with torch.cuda.device(dev):
            rc = lib.b200gsr_assemble_forward(num_groups, _group_table(raw), M, B, c_shs, c_scale, ptr(z_shs), ptr(z_scales),
                                              seed, *[ptr(o) for o in out], _lib.stream(dev))
        _lib.check(rc, "b200gsr_assemble_forward")
        ctx.meta = (num_groups, M, B, c_shs, c_scale, seed)
        ctx.noise = (z_shs, z_scales)
        ctx.save_for_backward(*[t for ts in raw for t in ts])
        return tuple(out)

    @staticmethod
    def backward(ctx, g_means, g_opac, g_scales, g_rots, g_shs):
        num_groups, M, B, c_shs, c_scale, seed = ctx.meta
        z_shs, z_scales = ctx.noise
        saved = ctx.saved_tensors
        raw = [list(saved[6 * k:6 * k + 6]) for k in range(num_groups)]
        dev = raw[0][0].device
        P = sum(int(ts[0].shape[0]) for ts in raw)
        shapes = [(P, 3), (P, 1), (B, P, 3), (P, 4), (B, P, M, 3)]
        gin = [torch.zeros(s, device=dev) if g is None else _lib.prepare(g.detach())
               for g, s in zip((g_means, g_opac, g_scales, g_rots, g_shs), shapes)]
        grads = [[torch.empty_like(t) for t in ts] for ts in raw]
        garr = (_lib.GroupGrad * num_groups)()
        for k, ts in enumerate(grads):
            for name, t in zip(("xyz", "opacity", "scaling", "rotation", "f_dc", "f_rest"), ts):
                setattr(garr[k], name, t.data_ptr() if t.numel() else None)
        lib, ptr = _lib.load(), _lib.ptr
        with torch.cuda.device(dev):
            rc = lib.b200gsr_assemble_backward(num_groups, _group_table(raw), garr, M, B, c_shs, c_scale, ptr(z_shs),
                                               ptr(z_scales), seed, *[ptr(g) for g in gin], _lib.stream(dev))
        _lib.check(rc, "b200gsr_assemble_backward")
        return (None,) * 8 + tuple(t for ts in grads for t in ts)


def assemble_scene(groups: Sequence, shs_aug: bool = True, scale_aug: bool = True, noise: str = "torch",
                   seed: int | None = None, generator: torch.Generator | None = None,
                   z_shs: torch.Tensor | None = None, z_scales: torch.Tensor | None = None, views: int = 1):
    """-> (means3D[P,3], opacities[P,1], scales[P,3], rotations[P,4], shs[P,M,3]) ready for
    GaussianRasterizer, differentiable w.r.t. every group's raw leaves.  z_shs [P,M,3] / z_scales [P,3]:
    explicit standard-normal draws (noise="torch" only; drawn with torch.randn when omitted).

    views = B > 1: the B views of one training step in ONE pass over the raw parameters: returns
    scales [B,P,3] and shs [B,P,M,3] (an independently augmented copy per view; index them per view for
    rasterize_views), means3D / opacities / rotations once; the backward sums the per-view gradients in the
    kernel.  With noise="torch" the draws follow the reference's order view by view (shs, then scales)."""
    if not 1 <= len(groups) <= _lib.MAX_GROUPS:
        raise ValueError(f"need 1..{_lib.MAX_GROUPS} groups")
    if noise not in ("torch", "fused"):
        raise ValueError("noise must be 'torch' or 'fused'")
    flat = [_get(g, name) for g in groups for name in _FIELDS]
    dev = flat[0].device
    if dev.type != "cuda":
        raise RuntimeError("assemble_scene (b200gsr): parameters must be CUDA tensors; there is no CPU fallback")
    M = 1 + int(_get(groups[0], "_features_rest").shape[1])
    P = sum(int(_get(g, "_xyz").shape[0]) for g in groups)
    B = int(views)
    if not 1 <= B <= _lib.MAX_VIEWS:
        raise ValueError(f"views must be in 1..{_lib.MAX_VIEWS}")
    if noise == "torch":
        # the reference's order of draws: per view, randn_like(shs) first, then randn_like(scales)
        zs, zc = [], []
        for v in range(B):
            if shs_aug and z_shs is None:
                zs.append(torch.randn(P, M, 3, device=dev, generator=generator))
            if scale_aug and z_scales is None:
                zc.append(torch.randn(P, 3, device=dev, generator=generator))
        if zs:
            z_shs = zs[0] if B == 1 else torch.stack(zs)
        if zc:
            z_scales = zc[0] if B == 1 else torch.stack(zc)
        z_shs = _lib.prepare(z_shs.detach()) if shs_aug else None
        z_scales = _lib.prepare(z_scales.detach()) if scale_aug else None
        if (z_shs is not None and z_shs.numel() != B * P * M * 3) or (z_scales is not None and z_scales.numel() != B * P * 3):
            raise ValueError("noise tensors must hold one draw per view and element")
        seed = 0
    else:
        z_shs = z_scales = None
        if seed is None:
            cpu_gen = generator if generator is not None and generator.device.type == "cpu" else None
            seed = int(torch.randint(0, 2 ** 62, (1,), generator=cpu_gen).item())
    m, o, sc, r, sh = _Assemble.apply(len(groups), M, B, NOISE_COEF if shs_aug else 0.0, NOISE_COEF if scale_aug else 0.0,
                                      z_shs, z_scales, int(seed), *flat)
    return (m, o, sc[0], r, sh[0]) if B == 1 else (m, o, sc, r, sh)


# ------------------------------------------------------------------------------------------------------------------
# render_scene: the views of a training step rendered straight from the raw parameter groups (include/b200gsr_scene.h)
# ------------------------------------------------------------------------------------------------------------------
def _view_flags(flag, B: int, name: str):
    """A bool, or a sequence of B bools (the reference's per-view ``random.random() < ratio`` outcomes) -> B bools."""
    if isinstance(flag, (bool, int)) or getattr(flag, "ndim", None) == 0:      # also numpy / tensor scalars
        return (bool(flag),) * B
    flags = tuple(bool(f) for f in flag)
    if len(flags) != B:
        raise ValueError(f"{name}: expected a bool or {B} per-view bools, got {len(flags)}")
    return flags


def _scene_groups(groups: Sequence):
    """-> (flat raw leaves in _FIELDS order per group, M, P).  Refuses anything the kernels cannot take (the device
    last, after every shape check)."""
    if not 1 <= len(groups) <= _lib.MAX_GROUPS:
        raise ValueError(f"need 1..{_lib.MAX_GROUPS} groups")
    flat = [_get(g, name) for g in groups for name in _FIELDS]
    Ms = {1 + int(_get(g, "_features_rest").shape[1]) for g in groups}
    if len(Ms) != 1:
        raise ValueError(f"render_scene: every group must have the same number of SH coefficients, got {sorted(Ms)}")
    M = Ms.pop()
    if M > 16:
        raise ValueError(f"render_scene: M={M} SH coefficients per channel, at most 16 (degree 3)")
    P = sum(int(_get(g, "_xyz").shape[0]) for g in groups)
    return flat, M, P


def _refuse_reserved(groups: Sequence):
    if any(getattr(g, "_reserved_rows", False) for g in groups):
        raise TypeError("render_scene: a ReservedGroup holds dead rows past its live count; render group.rows() (the "
                        "live prefixes) eagerly, or replay it with StepGraph")


def _check_device(flat):
    if any(t.device.type != "cuda" for t in flat):
        raise RuntimeError("render_scene (b200gsr): parameters must be CUDA tensors; there is no CPU fallback")
    if len({t.device for t in flat}) != 1:
        raise ValueError("render_scene: every group must live on one device")


def _check_settings(settings):
    B = len(settings)
    if not 1 <= B <= _lib.MAX_VIEWS:
        raise ValueError(f"need 1..{_lib.MAX_VIEWS} views")
    H, W = int(settings[0].image_height), int(settings[0].image_width)
    for s in settings:
        if int(s.image_height) != H or int(s.image_width) != W:
            raise ValueError("render_scene: all views must share the image size")
        if bool(s.score_flag):
            raise ValueError("render_scene: score_flag is not supported; use dreamscene_b200.filtering for the "
                             "important score")
    return B, H, W


def _frozen_mask(frozen, num_groups: int, who: str) -> int:
    """None (nothing frozen) or one bool per group -> the bit mask of the frozen groups (bit g = group g)."""
    if frozen is None:
        return 0
    flags = [bool(f) for f in frozen]
    if len(flags) != num_groups:
        raise ValueError(f"{who}: frozen must hold one bool per group ({num_groups}), got {len(flags)}")
    return sum(1 << g for g, f in enumerate(flags) if f)


def _densify_stats(densify_stats, groups: Sequence, frozen_mask: int, who: str):
    """None, or one entry per group - None or (xyz_gradient_accum, denom, max_radii2D or None) - -> a tuple of the
    validated entries (the tensors themselves: they are updated in place), or None when no group gathers."""
    if densify_stats is None:
        return None
    entries = list(densify_stats)
    if len(entries) != len(groups):
        raise ValueError(f"{who}: densify_stats must hold one entry per group ({len(groups)}), got {len(entries)}")
    out = []
    for g, (grp, e) in enumerate(zip(groups, entries)):
        if e is None:
            out.append(None)
            continue
        if len(e) != 3 or e[0] is None or e[1] is None:
            raise ValueError(f"{who}: densify_stats[{g}] must be (xyz_gradient_accum, denom, max_radii2D or None)")
        if (frozen_mask >> g) & 1:
            raise ValueError(f"{who}: densify_stats[{g}] gathers statistics for frozen group {g}; the reference gathers "
                             "them for the trained groups only")
        xyz = _get(grp, "_xyz")
        n = int(xyz.shape[0])
        for name, t in zip(("xyz_gradient_accum", "denom", "max_radii2D"), e):
            if t is None:
                continue
            if not torch.is_tensor(t) or t.dtype != torch.float32 or not t.is_contiguous():
                raise ValueError(f"{who}: densify_stats[{g}] {name} must be a contiguous float32 tensor")
            if t.numel() != n:
                raise ValueError(f"{who}: densify_stats[{g}] {name} has {t.numel()} elements, group {g} has {n} rows")
            if t.device != xyz.device:
                raise ValueError(f"{who}: densify_stats[{g}] {name} must be on the groups' device ({xyz.device})")
        out.append((e[0], e[1], e[2]))
    return tuple(out) if any(e is not None for e in out) else None


def _stats_table(stats):
    """The b200gsr_group_stats records of _densify_stats' entries (NULL for None: no group gathers)."""
    if stats is None:
        return None
    arr = (_lib.GroupStats * len(stats))()
    for g, e in enumerate(stats):
        if e is not None:
            arr[g] = _lib.GroupStats(*[None if t is None else t.data_ptr() for t in e])
    return arr


class _RenderScene(torch.autograd.Function):
    @staticmethod
    def forward(ctx, settings, num_groups, M, c_shs, c_scale, seed, return_scales, frozen, stats, *flat):
        # flat = 6 raw leaves per group, then the B means2D ports (none when `stats` = (entries, view) is given
        # without them: then no screen-space gradient is stored at all)
        from . import rasterizer as R
        B = len(settings)
        raw = [[_lib.prepare(t.detach()) for t in flat[6 * k:6 * k + 6]] for k in range(num_groups)]
        dev = raw[0][0].device
        P = sum(int(ts[0].shape[0]) for ts in raw)
        H, W = int(settings[0].image_height), int(settings[0].image_width)
        with_backward = any(ctx.needs_input_grad)
        d = R._device_state(dev)
        capturing = torch.cuda.is_current_stream_capturing()
        if not capturing:
            d.resolve()
        keep: list = []
        lib, ptr = _lib.load(), _lib.ptr
        noise = ((C.c_float * B)(*c_shs), (C.c_float * B)(*c_scale))
        with torch.cuda.device(dev):
            Hs = _lib.stacked_height(B, H, W)
            bg_all = torch.stack([R._const(s.bg, dev).reshape(3) for s in settings]).contiguous()
            prm = (_lib.Params * B)(*[R._make_params(s, P, M, keep, dev, bg_all, v) for v, s in enumerate(settings)])
            table = _group_table(raw)
            color = torch.empty(3, Hs, W, dtype=torch.float32, device=dev)
            depth_alpha = torch.empty(2, Hs, W, dtype=torch.float32, device=dev)
            radii = torch.empty(B, P, dtype=torch.int32, device=dev)
            scales = torch.empty(B, P, 3, dtype=torch.float32, device=dev) if return_scales else None
            stream = _lib.stream(dev)
            det = R.deterministic_mode()

            def launch(cap, flags, scratch, saved, notify_ptr, seq):
                return lib.b200gsr_forward_scene(B, prm, num_groups, table, noise[0], noise[1], seed, ptr(scales),
                                                 ptr(color), ptr(depth_alpha), ptr(radii), ptr(scratch), scratch.numel(),
                                                 ptr(saved), saved.numel(), cap, flags, notify_ptr, seq, stream)

            saved, cap = R._issue_with_capacity(d, (B, P, H, W), B * P, Hs, W, with_backward, det, None, launch,
                                                capturing, stream.value)
        ctx.meta = (B, P, M, W, Hs, cap, with_backward, num_groups, seed, det, frozen)
        ctx.stats = stats
        ctx.ports = len(flat) - 6 * num_groups
        ctx.views = (prm, table, noise)   # reused by the backward; `keep` holds the device constants of `prm`
        ctx.keep = keep
        ctx.saved_buf = saved
        ctx.save_for_backward(radii, depth_alpha, *[t for ts in raw for t in ts])
        ctx.mark_non_differentiable(radii)
        ctx.set_materialize_grads(False)
        if scales is not None:
            return color, radii, depth_alpha, scales
        return color, radii, depth_alpha

    @staticmethod
    def backward(ctx, g_color, _g_radii, g_da, g_scales=None):
        B, P, M, W, Hs, cap, with_backward, num_groups, seed, det, frozen = ctx.meta
        stats = ctx.stats
        prm, table, noise = ctx.views
        radii, depth_alpha = ctx.saved_tensors[:2]
        leaves = ctx.saved_tensors[2:]
        raw = [list(leaves[6 * k:6 * k + 6]) for k in range(num_groups)]
        dev = radii.device
        if not with_backward:
            raise RuntimeError("b200gsr: backward through a forward that ran without gradient accumulators")
        # every row of a trainable group is written by view 0; a frozen group gets no gradient
        grads = [[None] * 6 if (frozen >> k) & 1 else [torch.empty_like(t) for t in ts] for k, ts in enumerate(raw)]
        d_means2D = torch.zeros(B, P, 3, dtype=torch.float32, device=dev) if ctx.ports else None
        if P > 0:
            g_color = torch.zeros(3, Hs, W, device=dev) if g_color is None else _lib.prepare(g_color)
            g_da = torch.zeros(2, Hs, W, device=dev) if g_da is None else _lib.prepare(g_da)
            g_scales = None if g_scales is None else _lib.prepare(g_scales)
            garr = (_lib.GroupGrad * num_groups)()
            for k, ts in enumerate(grads):
                for name, t in zip(("xyz", "opacity", "scaling", "rotation", "f_dc", "f_rest"), ts):
                    setattr(garr[k], name, t.data_ptr() if t is not None and t.numel() else None)
            lib, ptr = _lib.load(), _lib.ptr
            args = (B, prm, num_groups, table, garr, noise[0], noise[1], seed, ptr(g_scales), ptr(radii),
                    ptr(depth_alpha), ptr(g_color), ptr(g_da), ptr(ctx.saved_buf), ctx.saved_buf.numel(), cap,
                    ptr(d_means2D), _lib.BWD_DETERMINISTIC if det else 0)
            with torch.cuda.device(dev):
                if stats is not None:
                    name = "b200gsr_backward_scene_stats"
                    rc = lib.b200gsr_backward_scene_stats(*args, frozen, _stats_table(stats[0]), stats[1], _lib.stream(dev))
                elif frozen:
                    name = "b200gsr_backward_scene_frozen"
                    rc = lib.b200gsr_backward_scene_frozen(*args, frozen, _lib.stream(dev))
                else:
                    name = "b200gsr_backward_scene"
                    rc = lib.b200gsr_backward_scene(*args, _lib.stream(dev))
            _lib.check(rc, name)
        ports = tuple(d_means2D.unbind(0)) if ctx.ports else ()
        return (None,) * 9 + tuple(t for ts in grads for t in ts) + ports


def render_scene(groups: Sequence, settings_list: Sequence, *, shs_aug=True, scale_aug=True, seed: int | None = None,
                 generator: torch.Generator | None = None, means2D: Sequence[torch.Tensor] | None = None,
                 return_scales: bool = False, frozen: Sequence[bool] | None = None, densify_stats: Sequence | None = None,
                 stats_view: int = -1):
    """The B views of one training step rendered straight from the raw parameter groups: activations, augmentation
    and rasterization in one op (the reference's scene_render / object_render, scene_gaussian.py:673-893).

    groups        : as assemble_scene (at most MAX_GROUPS, every group with the same M).
    settings_list : 1..MAX_VIEWS GaussianRasterizationSettings of one image size, as rasterize_views (camera, bg,
                    sh_degree and scale_modifier may differ per view); score_flag must be False.
    shs_aug / scale_aug : a bool, or B bools (the reference's per-view ``random.random() < ratio`` outcomes).
    seed / generator : the in-kernel Philox noise of assemble_scene(noise="fused"): for equal seeds the rasterizer
                    sees bit for bit the inputs of assemble_scene(groups, noise="fused", seed=seed, views=B).
    means2D       : optional B [P,3] tensors whose .grad receives the per-view screen-space gradient.
    frozen        : None, or one bool per group.  A frozen group is rendered as any other but trained by none of
                    the step's optimizers (the reference's stages that train one group): its leaves get None as their
                    gradient, its means2D rows get zeros, and the backward computes nothing for it.  The trainable
                    groups' gradients are those of the call without `frozen` (bit for bit in deterministic mode).
                    Explicit, not inferred from requires_grad: a group whose leaves need no gradient still feeds the
                    means2D gradients unless it is frozen.
    densify_stats : None, or one entry per group: None, or the reference's (xyz_gradient_accum, denom, max_radii2D or
                    None) of that group (float32, contiguous, one element per row).  The backward then also does the
                    reference's add_densification_stats for view `stats_view`, in place and inside the render
                    backward: for each row whose radius in that view is positive, accum += |screen-space gradient
                    [:2]|, denom += 1, max_radii2D = max(max_radii2D, radius) - bit for bit what
                    densify.add_densification_stats does with that view's means2D gradient and radii.  A frozen group
                    gathers nothing (refused).  Each backward adds once: a second backward through the same forward
                    (retain_graph) adds a second time, as calling the reference twice would.  Without `means2D` the
                    backward then stores no screen-space gradient at all (no [B,P,3] buffer).
    stats_view    : the view whose statistics are gathered: -1 (default) is the last view, B - 1 - the view whose
                    gradient the reference's `out` holds after its view loop.
    -> list of B (color[3,H,W], radii[P], depth_alpha[2,H,W]); with return_scales also the augmented scales
       [B,P,3] (differentiable, for the reference's scale loss).  Every trainable group's raw leaves get their
       gradients."""
    _refuse_reserved(groups)
    from . import parallel
    B, H, W = _check_settings(settings_list)
    shs_flags = _view_flags(shs_aug, B, "shs_aug")
    scale_flags = _view_flags(scale_aug, B, "scale_aug")
    flat, M, P = _scene_groups(groups)
    frozen_mask = _frozen_mask(frozen, len(groups), "render_scene")
    stats = _densify_stats(densify_stats, groups, frozen_mask, "render_scene")
    if densify_stats is not None:
        sv = int(stats_view)
        if not -1 <= sv < B:
            raise ValueError(f"render_scene: stats_view must be -1 (the last view) or in 0..{B - 1}, got {stats_view}")
        sv = B - 1 if sv == -1 else sv
    if parallel.reduction_active():
        raise RuntimeError("render_scene does not reduce gradients over ranks inside its backward; call "
                           "dreamscene_b200.parallel.all_reduce_gradients on the leaves after backward instead")
    _check_device(flat)
    dev = flat[0].device
    if means2D is None:
        # with densify_stats no port is needed: the backward then writes no screen-space gradient
        means2D = [] if densify_stats is not None else [torch.zeros(P, 3, device=dev) for _ in range(B)]
    if len(means2D) != B and not (densify_stats is not None and len(means2D) == 0):
        raise ValueError(f"means2D: expected {B} per-view tensors")
    if seed is None:
        cpu_gen = generator if generator is not None and generator.device.type == "cpu" else None
        seed = int(torch.randint(0, 2 ** 62, (1,), generator=cpu_gen).item())
    res = _RenderScene.apply(tuple(settings_list), len(groups), M,
                             tuple(NOISE_COEF if f else 0.0 for f in shs_flags),
                             tuple(NOISE_COEF if f else 0.0 for f in scale_flags), int(seed), bool(return_scales),
                             frozen_mask, None if densify_stats is None else (stats, sv), *flat, *means2D)
    color, radii, da = res[0], res[1], res[2]
    Hp = color.shape[1] // B
    outs = [(color[:, v * Hp:v * Hp + H, :], radii[v], da[:, v * Hp:v * Hp + H, :]) for v in range(B)]
    return (outs, res[3]) if return_scales else outs
