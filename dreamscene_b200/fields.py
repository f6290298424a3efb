"""The opacity field of a Gaussian group on a voxel grid, the reference's GaussianModel.extract_fields.

DreamScene's extract_fields (gs_renderer.py) loops over num_blocks^3 grid blocks in Python and, per block, builds
[points, Gaussians, 3] and [points, Gaussians, 6] tensors of every Gaussian near the block.  ``extract_fields(group)``
computes the same field with one pass of kernels (include/b200gsr_fields.h): a filter and normalisation pass, a
binning pass that lists every block's Gaussians in row order, and one CTA per block summing its grid points in
registers.  ``extract_fields_rgb(group)`` evaluates the group's colour field in the same pass: the opacity-weighted
mean of the Gaussians' view-independent colours, which mesh.extract_coloured_mesh carries onto a mesh.
"""
from __future__ import annotations

import ctypes as C
from typing import Tuple

import torch

from . import _lib
from . import scene as S

_LEAVES = ("_xyz", "_opacity", "_scaling", "_rotation")


def _check_group(group):
    S._refuse_reserved([group])
    leaves = [S._get(group, name) for name in _LEAVES]
    P = int(leaves[0].shape[0])
    shapes = [(P, 3), (P, 1), (P, 3), (P, 4)]
    for name, t, shape in zip(_LEAVES, leaves, shapes):
        if tuple(t.shape) != shape:
            raise ValueError(f"extract_fields: {name} has shape {tuple(t.shape)}, expected {shape}")
    if P == 0:
        raise ValueError("extract_fields: no Gaussian has opacity above 0.005 (the group is empty)")
    if any(t.device.type != "cuda" for t in leaves):
        raise ValueError("extract_fields (b200gsr): parameters must be CUDA tensors; there is no CPU fallback")
    if len({t.device for t in leaves}) != 1:
        raise ValueError("extract_fields: every leaf must live on one device")
    return leaves, P


def extract_fields(group, resolution: int = 128, num_blocks: int = 16,
                   relax_ratio: float = 1.5) -> Tuple[torch.Tensor, torch.Tensor, float]:
    """The reference's extract_fields(resolution, num_blocks, relax_ratio) of one Gaussian group.

    group       : a plain group with _xyz [P,3], _opacity [P,1], _scaling [P,3], _rotation [P,4] CUDA tensors (the
                  raw leaves, as render_scene takes them), or ReservedGroup.rows(); a ReservedGroup itself is refused.
    resolution  : R, grid points per axis, 1..1024.  resolution % (2 / num_blocks) must be 0, as the reference
                  asserts.
    num_blocks  : 1..R; the coordinates are cut into chunks of R // num_blocks points, the last one possibly shorter,
                  at most 32 chunks per axis.
    relax_ratio : how far, in blocks of 2 / num_blocks, a Gaussian's centre may lie outside a block and still reach it.
    -> (occ float32 CUDA [R,R,R], center float32 CUDA [3], scale float): the field and the normalisation the reference
       stores in self.center / self.scale; grid point (i, j, k) lies at world position
       center + (X[i], X[j], X[k]) / scale with X = torch.linspace(-1, 1, R).

    Rows with sigmoid(_opacity) > 0.005 are kept; center = (mn + mx) / 2 and scale = 1.8 / max(mx - mn) (in double)
    over their centres; the centres xyz' = (xyz - center) * scale and the standard deviations exp(_scaling) * scale
    are float32, as torch computes them.  A Gaussian belongs to a block when its normalised centre lies strictly
    inside the block's coordinate box widened by (2 / num_blocks) * relax_ratio on every side; a Gaussian outside that
    box adds nothing to the block's points, however large it is (the reference's rule).  These membership decisions
    are bit for bit those of torch's float32 evaluation of the reference.  occ[i,j,k] is the sum over the block's
    members of opacity * exp(-1/2 d^T Sigma^-1 d), with the reference's cofactor inverse (1e-24 added to the
    determinant) and weight 0 where that exponent is positive.  The sum runs in row order, in a different order
    from the reference's batches, so it agrees to a float32 reordering tolerance; it is the same bits on every call.

    Refused with ValueError: CPU tensors, bad sizes, no row passing the opacity filter, and kept centres that all
    coincide (the reference divides by zero).  The call waits for the device to read the normalisation back, so it
    cannot be captured into a CUDA graph.  No gradients."""
    return _evaluate(group, resolution, num_blocks, relax_ratio, None)


def extract_fields_rgb(group, resolution: int = 128, num_blocks: int = 16,
                       relax_ratio: float = 1.5) -> Tuple[torch.Tensor, torch.Tensor, torch.Tensor, float]:
    """extract_fields(group, resolution, num_blocks, relax_ratio) and the group's colour field on the same grid.

    group also needs _features_dc [P,1,3], the degree-0 SH coefficients, as a CUDA tensor on the leaves' device.
    -> (occ [R,R,R], rgb float32 CUDA [R,R,R,3], center [3], scale): occ, center and scale are bit for bit what
       extract_fields returns.  Each Gaussian's colour is c = clamp_min(_features_dc * SH_C0 + 0.5, 0), the reference's
       SH2RGB clamped at 0 as the renderer clamps it, in float32: the mean of its SH colour over all view directions,
       so the colour is view-independent.  rgb[i,j,k] = (sum of opacity * weight * c over the members occ sums, in
       the same order) / occ[i,j,k], 0 where occ is 0: a weighted mean of the member colours, so every value lies
       between the smallest and largest of them, up to rounding, where occ is not a tiny (subnormal-range) value.
       It is not clamped above 1.  The sums are float32 in row order, the same bits on every call
       (include/b200gsr_mesh_colour.h).

    Refused with ValueError: what extract_fields refuses, a missing or misshapen _features_dc, and grids with
    3 R^3 >= 2^31 (R above 894).  Waits for the device, as extract_fields does; no gradients."""
    return _evaluate(group, resolution, num_blocks, relax_ratio, "extract_fields_rgb")


def _features_dc(group, P, dev, what):
    try:
        dc = S._get(group, "_features_dc")
    except (KeyError, AttributeError):
        raise ValueError(f"{what}: the group has no _features_dc") from None
    if not isinstance(dc, torch.Tensor) or tuple(dc.shape) != (P, 1, 3):
        shape = tuple(dc.shape) if isinstance(dc, torch.Tensor) else type(dc).__name__
        raise ValueError(f"{what}: _features_dc has shape {shape}, expected {(P, 1, 3)}")
    if dc.device != dev:
        raise ValueError(f"{what}: _features_dc must live on the leaves' device {dev}")
    return dc


def _evaluate(group, resolution, num_blocks, relax_ratio, rgb_of):
    """The field of extract_fields and, when rgb_of names the caller, the colour field beside it."""
    resolution, num_blocks, relax_ratio = int(resolution), int(num_blocks), float(relax_ratio)
    if not 1 <= num_blocks <= resolution:
        raise ValueError(f"extract_fields: num_blocks must be in 1..resolution, got {num_blocks} for {resolution}")
    if resolution % (2 / num_blocks) != 0:
        raise ValueError(f"extract_fields: resolution {resolution} is not a multiple of the block size 2 / "
                         f"{num_blocks} (the reference asserts resolution % block_size == 0)")
    leaves, P = _check_group(group)
    dev = leaves[0].device
    dc = None if rgb_of is None else _features_dc(group, P, dev, rgb_of)
    coords = torch.linspace(-1, 1, resolution)          # torch's float32 coordinates, on the host
    lib = _lib.load()
    layout = _lib.FieldsLayout()
    cptr = C.c_void_p(coords.data_ptr())
    query = "b200gsr_fields_layout_query" if dc is None else "b200gsr_fields_rgb_layout_query"
    _lib.check(getattr(lib, query)(P, resolution, num_blocks, relax_ratio, cptr, C.byref(layout)), query, ValueError)
    with torch.no_grad(), torch.cuda.device(dev):
        xyz, opacity, scaling, rotation = [_lib.prepare(t.detach()) for t in leaves]
        occ = torch.empty((resolution,) * 3, dtype=torch.float32, device=dev)
        info = torch.empty(C.sizeof(_lib.FieldsInfo), dtype=torch.uint8, device=dev)
        scratch = torch.empty(layout.total, dtype=torch.uint8, device=dev)
        ptr = _lib.ptr
        if dc is None:
            _lib.check(lib.b200gsr_fields(P, ptr(xyz), ptr(opacity), ptr(scaling), ptr(rotation), resolution,
                                          num_blocks, relax_ratio, cptr, ptr(occ), ptr(info), ptr(scratch),
                                          scratch.numel(), _lib.stream(dev)), "b200gsr_fields", ValueError)
        else:
            dc = _lib.prepare(dc.detach())
            rgb = torch.empty((resolution,) * 3 + (3,), dtype=torch.float32, device=dev)
            _lib.check(lib.b200gsr_fields_rgb(P, ptr(xyz), ptr(opacity), ptr(scaling), ptr(rotation), ptr(dc),
                                              resolution, num_blocks, relax_ratio, cptr, ptr(occ), ptr(rgb), ptr(info),
                                              ptr(scratch), scratch.numel(), _lib.stream(dev)), "b200gsr_fields_rgb",
                       ValueError)
        res = _lib.FieldsInfo.from_buffer_copy(bytes(info.cpu().numpy()))
    if res.kept == 0:
        raise ValueError("extract_fields: no Gaussian has opacity above 0.005")
    if res.extent == 0:
        raise ValueError("extract_fields: every kept Gaussian has the same centre, so the field has no scale")
    if res.overflow:
        raise RuntimeError("extract_fields: the member lists overflowed their capacity")
    center = torch.tensor(list(res.center), dtype=torch.float32, device=dev)
    return (occ, center, float(res.scale)) if dc is None else (occ, rgb, center, float(res.scale))
