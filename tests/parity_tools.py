"""Parity measurement helpers shared by the GPU tests and tools/parity_stats.py.

Everything here is CHECKER code: it drives the CUDA product through its public surface and compares
with the CPU oracle (oracle/splat_ref.py).  Three things the plain image comparison cannot do:

* forward_stats       - the measured outlier statistics (how many values differ by more than the
                        north-star tolerance 1e-4, and by how much) instead of a pass/fail;
* sample_tiles        - a deterministic, list-length-stratified sample of non-empty tiles;
* oracle_backward_on_tiles - the COMPLETE parameter gradient of a loss whose incoming image gradients
                        are non-zero only on the sampled tiles: the oracle blends just those tiles
                        (fp64 on the fp32 pair lists), the CUDA path back-propagates the masked
                        gradients through the whole frame, and the two full [P, ...] gradients are
                        comparable at sizes (1M Gaussians / 1024^2) where the oracle cannot render the
                        frame.  Tiles are blended in small groups so autograd never holds more than a
                        few tiles' intermediates.
"""
from __future__ import annotations

import numpy as np
import torch

from oracle import splat_ref as O
from tests import util_scene as U

FWD_ATOL = 1e-4   # north_star: forward RGB/depth/alpha within 1e-4 abs


def forward_stats(cu_color, cu_da, ref_color, ref_da, cu_nc=None, ref_nc=None, mask=None):
    """-> {channel: {n, n_bad, frac_bad, max_abs, p999}} for colour, depth and T (+ n_contrib mismatch
    rate).  `mask` [H,W] bool restricts the comparison to the sampled tiles."""
    out = {}
    m = None if mask is None else mask.reshape(-1)
    chans = {"color": (cu_color.detach().cpu().float(), ref_color.detach().float()),
             "depth": (cu_da[0].detach().cpu().float(), ref_da[0].detach().float()),
             "T": (cu_da[1].detach().cpu().float(), ref_da[1].detach().float())}
    for name, (a, b) in chans.items():
        d = (a - b).abs()
        d = d.reshape(3, -1)[:, m].reshape(-1) if (m is not None and d.dim() == 3) else (d.reshape(-1)[m] if m is not None else d.reshape(-1))
        n = d.numel()
        bad = int((d > FWD_ATOL).sum())
        out[name] = {"n": n, "n_bad": bad, "frac_bad": bad / max(n, 1), "max_abs": float(d.max()) if n else 0.0,
                     "p999": float(torch.quantile(d.double(), 0.999)) if 0 < n <= 16_000_000 else None}
    if cu_nc is not None and ref_nc is not None:
        a = np.asarray(cu_nc).reshape(-1).astype(np.int64)
        b = np.asarray(ref_nc).reshape(-1).astype(np.int64)
        if m is not None:
            a, b = a[m.numpy()], b[m.numpy()]
        out["n_contrib"] = {"n": int(a.size), "n_mismatch": int((a != b).sum()),
                            "frac_mismatch": float((a != b).mean()) if a.size else 0.0,
                            "max_abs": int(np.abs(a - b).max()) if a.size else 0}
    return out


def sample_tiles(ranges, count):
    """`count` non-empty tiles, evenly spaced over the tiles ordered by list length (longest first)."""
    n = ranges[:, 1] - ranges[:, 0]
    order = np.argsort(-n, kind="stable")
    nonempty = int((n > 0).sum())
    if nonempty == 0:
        return []
    pos = np.unique(np.linspace(0, nonempty - 1, min(count, nonempty)).round().astype(np.int64))
    return [int(order[p]) for p in pos]


def tile_mask(tiles, H, W):
    gx = (W + 15) // 16
    m = torch.zeros(H, W, dtype=torch.bool)
    for t in tiles:
        ty, tx = divmod(int(t), gx)
        m[ty * 16:ty * 16 + 16, tx * 16:tx * 16 + 16] = True
    return m


def oracle_lists(sc, cam, deg, scale_modifier=1.0):
    """fp32 per-Gaussian stage + binning/sort (bit-exact integers) without blending anything.  The
    returned decisions also hold the fp32 EWA-clamp and colour-clamp flags for an fp64 replay."""
    S = U.oracle_settings(cam, deg, scale_modifier=scale_modifier)
    with torch.no_grad():
        pre = O.preprocess(S, sc["means3D"], sc["opacities"], shs=sc["shs"], scales=sc["scales"],
                           rotations=sc["rotations"])
        keys, pl, ranges = O.bin_and_sort(pre, S)
    dec = dict(visible=pre["visible"], radii=pre["radii"], rect=pre["rect"], touched=pre["touched"],
               point_list=pl, ranges=ranges, in_x=pre["in_x"], in_y=pre["in_y"], clamped=pre["clamped"])
    return S, pre, keys, pl, ranges, dec


def record_blend_decisions(pre32, dec, S, tiles):
    """fp32 blend pass over `tiles` that records the per-(entry, pixel) blend decisions (see
    oracle.splat_ref.composite) for replay by the fp64 gradient evaluation."""
    rec = {}
    with torch.no_grad():
        O.composite(pre32, dec["point_list"], dec["ranges"], S, tiles=tiles, record_blend=rec)
    return rec


def oracle_backward_on_tiles(sc, cam, deg, tiles, gc, gd, dec, dtype=torch.float64, group=6, blend=None):
    """Complete parameter gradients of  sum(color*gc) + sum(depth_alpha*gd)  where gc/gd are already
    zero outside `tiles`; blending in `dtype` on the fp32 decisions `dec` (and, when `blend` holds the
    recorded fp32 per-pixel blend decisions, on exactly those as well)."""
    S = U.oracle_settings(cam, deg)
    names = ("means3D", "opacities", "shs", "scales", "rotations")
    t = {k: sc[k].detach().clone().requires_grad_(True) for k in names}
    m2d = torch.zeros(sc["means3D"].shape[0], 3, requires_grad=True)
    pre = O.preprocess(S, t["means3D"].to(dtype), t["opacities"].to(dtype), shs=t["shs"].to(dtype),
                       scales=t["scales"].to(dtype), rotations=t["rotations"].to(dtype),
                       means2D=m2d.to(dtype), dtype=dtype, decisions=dec)
    keys = ["px", "py", "opacity", "rgb", "depth"]
    mid = {k: pre[k].detach().requires_grad_(True) for k in keys}
    con = [c.detach().requires_grad_(True) for c in pre["conic"]]
    pre2 = dict(pre); pre2.update(mid); pre2["conic"] = tuple(con)
    leaves = [mid[k] for k in keys] + con
    acc = [torch.zeros_like(x) for x in leaves]
    gc, gd = gc.to(dtype), gd.to(dtype)
    tiles = list(tiles)
    for i in range(0, len(tiles), group):
        color, da, _, _ = O.composite(pre2, dec["point_list"], dec["ranges"], S, dtype, tiles=tiles[i:i + group],
                                      replay_blend=blend)
        loss = (color * gc).sum() + (da * gd).sum()
        g = torch.autograd.grad(loss, leaves, allow_unused=True)
        for a, gi in zip(acc, g):
            if gi is not None:
                a += gi
    outs = [pre[k] for k in keys] + list(pre["conic"])
    torch.autograd.backward(outs, acc)
    grads = {k: v.grad.detach() for k, v in t.items()}
    grads["means2D"] = m2d.grad.detach()
    return grads


def cuda_forward_backward(sc, cam, deg, gc, gd, device=None, score=False):
    """Public surface -> C ABI -> kernels.  Returns images, radii, gradients (CPU tensors) and state."""
    from dreamscene_b200 import GaussianRasterizer
    dev = torch.device("cuda", torch.cuda.current_device()) if device is None else device
    S = U.cuda_settings(cam, deg, device=dev, score=score)
    names = ("means3D", "opacities", "shs", "scales", "rotations")
    t = {k: sc[k].detach().to(dev).requires_grad_(True) for k in names}
    m2d = torch.zeros(sc["means3D"].shape[0], 3, device=dev, requires_grad=True)
    out = GaussianRasterizer(S)(means3D=t["means3D"], means2D=m2d, opacities=t["opacities"], shs=t["shs"],
                                scales=t["scales"], rotations=t["rotations"])
    color, radii, da = out[-3], out[-2], out[-1]
    torch.autograd.backward([color, da], [gc.to(dev), gd.to(dev)])
    torch.cuda.synchronize(dev)
    grads = {k: v.grad.detach().cpu() for k, v in t.items()}
    grads["means2D"] = m2d.grad.detach().cpu()
    return dict(color=color.detach().cpu(), depth_alpha=da.detach().cpu(), radii=radii.cpu(), grads=grads,
                score=out[0].detach().cpu() if score else None)


def grad_errors(cu_grads, ref_grads):
    """Norm-wise relative error per parameter (the north-star's 1e-3 rel) + the largest element error
    relative to the gradient's RMS over touched entries."""
    out = {}
    for k, r in ref_grads.items():
        a, b = cu_grads[k].double(), r.double()
        nz = b != 0
        rms = float(b[nz].pow(2).mean().sqrt()) if bool(nz.any()) else 0.0
        out[k] = {"rel_l2": float((a - b).norm() / b.norm().clamp_min(1e-300)),
                  "max_abs_over_rms": float((a - b).abs().max() / rms) if rms > 0 else 0.0,
                  "nonzero": int(nz.sum())}
    return out
