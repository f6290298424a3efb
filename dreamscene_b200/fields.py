"""The opacity field of a Gaussian group on a voxel grid, the reference's GaussianModel.extract_fields.

DreamScene's extract_fields (gs_renderer.py) loops over num_blocks^3 grid blocks in Python and, per block, builds
[points, Gaussians, 3] and [points, Gaussians, 6] tensors of every Gaussian near the block.  ``extract_fields(group)``
computes the same field with one pass of kernels (include/b200gsr_fields.h): a filter and normalisation pass, a
binning pass that lists every block's Gaussians in row order, and one CTA per block summing its grid points in
registers.
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
    resolution, num_blocks, relax_ratio = int(resolution), int(num_blocks), float(relax_ratio)
    if not 1 <= num_blocks <= resolution:
        raise ValueError(f"extract_fields: num_blocks must be in 1..resolution, got {num_blocks} for {resolution}")
    if resolution % (2 / num_blocks) != 0:
        raise ValueError(f"extract_fields: resolution {resolution} is not a multiple of the block size 2 / "
                         f"{num_blocks} (the reference asserts resolution % block_size == 0)")
    leaves, P = _check_group(group)
    dev = leaves[0].device
    coords = torch.linspace(-1, 1, resolution)          # torch's float32 coordinates, on the host
    lib = _lib.load()
    layout = _lib.FieldsLayout()
    cptr = C.c_void_p(coords.data_ptr())
    _lib.check(lib.b200gsr_fields_layout_query(P, resolution, num_blocks, relax_ratio, cptr, C.byref(layout)),
               "b200gsr_fields_layout_query", ValueError)
    with torch.no_grad(), torch.cuda.device(dev):
        xyz, opacity, scaling, rotation = [_lib.prepare(t.detach()) for t in leaves]
        occ = torch.empty((resolution,) * 3, dtype=torch.float32, device=dev)
        info = torch.empty(C.sizeof(_lib.FieldsInfo), dtype=torch.uint8, device=dev)
        scratch = torch.empty(layout.total, dtype=torch.uint8, device=dev)
        ptr = _lib.ptr
        _lib.check(lib.b200gsr_fields(P, ptr(xyz), ptr(opacity), ptr(scaling), ptr(rotation), resolution, num_blocks,
                                      relax_ratio, cptr, ptr(occ), ptr(info), ptr(scratch), scratch.numel(),
                                      _lib.stream(dev)), "b200gsr_fields", ValueError)
        res = _lib.FieldsInfo.from_buffer_copy(bytes(info.cpu().numpy()))
    if res.kept == 0:
        raise ValueError("extract_fields: no Gaussian has opacity above 0.005")
    if res.extent == 0:
        raise ValueError("extract_fields: every kept Gaussian has the same centre, so the field has no scale")
    if res.overflow:
        raise RuntimeError("extract_fields: the member lists overflowed their capacity")
    return occ, torch.tensor(list(res.center), dtype=torch.float32, device=dev), float(res.scale)
