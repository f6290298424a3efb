"""The reference's GaussianModel.extract_fields (gs_renderer.py) and its gaussian_3d_coeff restated in torch, with the
same operations in the same order.  The checker of dreamscene_b200.fields.extract_fields; not product code.

extract_fields(group, ..., dtype=torch.float64) keeps the float32 decisions (the opacity filter, the normalisation
and the block memberships, so both evaluations sum the same Gaussians at every point) and evaluates the centres, the
covariances, the weights and the sums in float64 from the raw leaves: the yardstick both float32 evaluations are
measured against.
"""
from __future__ import annotations

import torch


def gaussian_3d_coeff(xyzs, covs, return_power=False):
    """Weights exp(power) of offsets xyzs [N,3] under covariances covs [N,6] (the upper triangle a b c / d e / f):
    power = -1/2 d^T Sigma^-1 d with the cofactor inverse and 1e-24 added to the determinant, set to -1e10 where > 0."""
    x, y, z = xyzs[:, 0], xyzs[:, 1], xyzs[:, 2]
    a, b, c, d, e, f = covs.unbind(1)
    inv_det = 1 / (a * d * f + 2 * e * c * b - e**2 * a - c**2 * d - b**2 * f + 1e-24)
    inv_a = (d * f - e**2) * inv_det
    inv_b = (e * c - b * f) * inv_det
    inv_c = (e * b - c * d) * inv_det
    inv_d = (a * f - c**2) * inv_det
    inv_e = (b * c - e * a) * inv_det
    inv_f = (a * d - b**2) * inv_det
    power = -0.5 * (x**2 * inv_a + y**2 * inv_d + z**2 * inv_f) - x * y * inv_b - x * z * inv_c - y * z * inv_e
    raw = power.clone()
    power[power > 0] = -1e10
    w = torch.exp(power)
    return (w, raw) if return_power else w


def build_rotation(r):
    norm = torch.sqrt(r[:, 0] * r[:, 0] + r[:, 1] * r[:, 1] + r[:, 2] * r[:, 2] + r[:, 3] * r[:, 3])
    q = r / norm[:, None]
    R = torch.zeros((q.size(0), 3, 3), dtype=r.dtype, device=r.device)
    r, x, y, z = q[:, 0], q[:, 1], q[:, 2], q[:, 3]
    R[:, 0, 0] = 1 - 2 * (y * y + z * z)
    R[:, 0, 1] = 2 * (x * y - r * z)
    R[:, 0, 2] = 2 * (x * z + r * y)
    R[:, 1, 0] = 2 * (x * y + r * z)
    R[:, 1, 1] = 1 - 2 * (x * x + z * z)
    R[:, 1, 2] = 2 * (y * z - r * x)
    R[:, 2, 0] = 2 * (x * z - r * y)
    R[:, 2, 1] = 2 * (y * z + r * x)
    R[:, 2, 2] = 1 - 2 * (x * x + y * y)
    return R


def covariance(stds, rotation):
    """strip_symmetric(L L^T), L = R(rotation) diag(stds): the reference's build_covariance_from_scaling_rotation."""
    L = torch.zeros((stds.shape[0], 3, 3), dtype=stds.dtype, device=stds.device)
    for i in range(3):
        L[:, i, i] = stds[:, i]
    L = build_rotation(rotation) @ L
    S = L @ L.transpose(1, 2)
    return torch.stack([S[:, 0, 0], S[:, 0, 1], S[:, 0, 2], S[:, 1, 1], S[:, 1, 2], S[:, 2, 2]], dim=1)


def _leaf(group, name):
    return group[name] if isinstance(group, dict) else getattr(group, name)


def normalise(group):
    """Steps 1-3 in float32 -> dict(mask [P] bool, xyz [K,3] normalised centres, opacity [K,1], center [3],
    scale (Python float))."""
    opacities = torch.sigmoid(_leaf(group, "_opacity"))
    mask = (opacities > 0.005).squeeze(1)
    xyzs = _leaf(group, "_xyz")[mask]
    mn, mx = xyzs.amin(0), xyzs.amax(0)
    center = (mn + mx) / 2
    scale = 1.8 / (mx - mn).amax().item()
    return dict(mask=mask, xyz=(xyzs - center) * scale, opacity=opacities[mask], center=center, scale=scale)


def chunks(resolution, num_blocks):
    """(first index, coordinates) of every chunk of torch.linspace(-1, 1, resolution) on one axis (float32, CPU)."""
    block_size = 2 / num_blocks
    assert resolution % block_size == 0
    split_size = resolution // num_blocks
    X = torch.linspace(-1, 1, resolution).split(split_size)
    return [(k * split_size, xs) for k, xs in enumerate(X)]


def block_boxes(resolution, num_blocks, relax_ratio, device):
    """{(xi, yi, zi): (vmin [3], vmax [3])} float32 on `device`, as the reference widens each block's points."""
    block_size = 2 / num_blocks
    X = chunks(resolution, num_blocks)
    out = {}
    for xi, (_, xs) in enumerate(X):
        for yi, (_, ys) in enumerate(X):
            for zi, (_, zs) in enumerate(X):
                pts = _points(xs, ys, zs).to(device)
                vmin, vmax = pts.amin(0), pts.amax(0)
                vmin -= block_size * relax_ratio
                vmax += block_size * relax_ratio
                out[(xi, yi, zi)] = (vmin, vmax)
    return out


def _points(xs, ys, zs):
    xx, yy, zz = torch.meshgrid(xs, ys, zs, indexing="ij")
    return torch.cat([xx.reshape(-1, 1), yy.reshape(-1, 1), zz.reshape(-1, 1)], dim=-1)


def member_counts(group, resolution=128, num_blocks=16, relax_ratio=1.5):
    """Gaussians per block [C,C,C] int64 (CPU), by the reference's in-block test on the float32 centres."""
    n = normalise(group)
    C = len(chunks(resolution, num_blocks))
    out = torch.zeros(C, C, C, dtype=torch.int64)
    for (xi, yi, zi), (vmin, vmax) in block_boxes(resolution, num_blocks, relax_ratio, n["xyz"].device).items():
        out[xi, yi, zi] = int(((n["xyz"] < vmax).all(-1) & (n["xyz"] > vmin).all(-1)).sum())
    return out


def extract_fields(group, resolution=128, num_blocks=16, relax_ratio=1.5, dtype=torch.float32, blocks=None):
    """-> (occ [R,R,R] of `dtype` on the leaves' device, center float32 [3], scale).  blocks: an iterable of
    (xi, yi, zi) to evaluate (the others stay 0), or None for all."""
    n = normalise(group)
    mask, xyzs, opacities = n["mask"], n["xyz"], n["opacity"]
    device = xyzs.device
    rotation = _leaf(group, "_rotation")[mask]
    if dtype == torch.float32:
        stds = torch.exp(_leaf(group, "_scaling"))[mask] * n["scale"]
        gxyz, opas = xyzs, opacities
    else:
        center = n["center"].to(dtype)
        gxyz = (_leaf(group, "_xyz")[mask].to(dtype) - center) * n["scale"]
        stds = torch.exp(_leaf(group, "_scaling")[mask].to(dtype)) * n["scale"]
        opas = torch.sigmoid(_leaf(group, "_opacity")[mask].to(dtype))
        rotation = rotation.to(dtype)
    covs = covariance(stds, rotation)
    occ = torch.zeros([resolution] * 3, dtype=dtype, device=device)
    X = chunks(resolution, num_blocks)
    boxes = block_boxes(resolution, num_blocks, relax_ratio, device)
    wanted = None if blocks is None else set(map(tuple, blocks))
    for (xi, yi, zi), (vmin, vmax) in boxes.items():
        if wanted is not None and (xi, yi, zi) not in wanted:
            continue
        (x0, xs), (y0, ys), (z0, zs) = X[xi], X[yi], X[zi]
        member = (xyzs < vmax).all(-1) & (xyzs > vmin).all(-1)
        if not member.any():
            continue
        pts = _points(xs, ys, zs).to(device=device, dtype=dtype)
        m_xyz, m_cov, m_opa = gxyz[member], covs[member], opas[member].view(1, -1)
        g_pts = pts.unsqueeze(1).repeat(1, m_cov.shape[0], 1) - m_xyz.unsqueeze(0)
        g_covs = m_cov.unsqueeze(0).repeat(pts.shape[0], 1, 1)
        val = 0
        for start in range(0, g_covs.shape[1], 1024):
            end = min(start + 1024, g_covs.shape[1])
            w = gaussian_3d_coeff(g_pts[:, start:end].reshape(-1, 3), g_covs[:, start:end].reshape(-1, 6))
            val += (m_opa[:, start:end] * w.reshape(pts.shape[0], -1)).sum(-1)
        occ[x0:x0 + len(xs), y0:y0 + len(ys), z0:z0 + len(zs)] = val.reshape(len(xs), len(ys), len(zs))
    return occ, n["center"], n["scale"]


# ---- the colour field of include/b200gsr_mesh_colour.h (dreamscene_b200.fields.extract_fields_rgb) ----------------
SH_C0 = 0.28209479177387814          # the reference's utils/sh_utils.C0


def sh2rgb(features_dc):
    """Step 1: clamp_min(SH2RGB(_features_dc), 0) of [P,1,3] -> [P,3] float32, torch's float32 multiply by the Python
    scalar, then its add, then the clamp (which keeps NaN)."""
    return torch.clamp_min(features_dc.float()[:, 0] * SH_C0 + 0.5, 0)


def extract_fields_rgb(group, resolution=128, num_blocks=16, relax_ratio=1.5, dtype=torch.float32, blocks=None):
    """Step 2 beside extract_fields: -> (occ [R,R,R], rgb [R,R,R,3], both of `dtype`, center float32 [3], scale).

    The same members, boxes and weights as extract_fields; rgb = (sum of opacity * weight * colour) / occ, 0 where
    occ is 0.  The colours are step 1's float32 values in either dtype; with float64 the products and sums are float64.
    blocks: an iterable of (xi, yi, zi) to evaluate (the others stay 0), or None for all."""
    n = normalise(group)
    mask, xyzs, opacities = n["mask"], n["xyz"], n["opacity"]
    device = xyzs.device
    rotation = _leaf(group, "_rotation")[mask]
    colours = sh2rgb(_leaf(group, "_features_dc"))[mask].to(dtype)
    if dtype == torch.float32:
        stds = torch.exp(_leaf(group, "_scaling"))[mask] * n["scale"]
        gxyz, opas = xyzs, opacities
    else:
        gxyz = (_leaf(group, "_xyz")[mask].to(dtype) - n["center"].to(dtype)) * n["scale"]
        stds = torch.exp(_leaf(group, "_scaling")[mask].to(dtype)) * n["scale"]
        opas = torch.sigmoid(_leaf(group, "_opacity")[mask].to(dtype))
        rotation = rotation.to(dtype)
    covs = covariance(stds, rotation)
    occ = torch.zeros([resolution] * 3, dtype=dtype, device=device)
    num = torch.zeros([resolution] * 3 + [3], dtype=dtype, device=device)
    X = chunks(resolution, num_blocks)
    wanted = None if blocks is None else set(map(tuple, blocks))
    for (xi, yi, zi), (vmin, vmax) in block_boxes(resolution, num_blocks, relax_ratio, device).items():
        if wanted is not None and (xi, yi, zi) not in wanted:
            continue
        (x0, xs), (y0, ys), (z0, zs) = X[xi], X[yi], X[zi]
        member = (xyzs < vmax).all(-1) & (xyzs > vmin).all(-1)
        if not member.any():
            continue
        pts = _points(xs, ys, zs).to(device=device, dtype=dtype)
        d = pts.unsqueeze(1) - gxyz[member].unsqueeze(0)                                  # [points, members, 3]
        w = gaussian_3d_coeff(d.reshape(-1, 3), covs[member].repeat(len(pts), 1)).view(len(pts), -1)
        ow = opas[member].view(1, -1) * w
        sl = (slice(x0, x0 + len(xs)), slice(y0, y0 + len(ys)), slice(z0, z0 + len(zs)))
        occ[sl] = ow.sum(-1).view(len(xs), len(ys), len(zs))
        num[sl] = (ow @ colours[member]).view(len(xs), len(ys), len(zs), 3)
    rgb = torch.where(occ.unsqueeze(-1) > 0, num / occ.unsqueeze(-1), torch.zeros_like(num))
    return occ, rgb, n["center"], n["scale"]
