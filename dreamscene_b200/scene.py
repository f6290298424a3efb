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
"""
from __future__ import annotations

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
