"""Pure-PyTorch CPU restatement of the differentiable 3D-Gaussian rasterizer that
DreamScene imports as ``diff_gaussian_rasterization``.

THIS FILE IS TEST INFRASTRUCTURE (the parity oracle and the "pure-PyTorch CPU splat"
baseline of BASELINE.json config 1).  The product never imports it.

Parity pinning
--------------
The CUDA source of the reference op (DreamScene-Project/comp-diff-gaussian-rasterization,
unpinned HEAD, /root/reference/README.md:47,50) is NOT vendored under /root/reference
(/root/reference/.gitignore:6) and cannot be built or run here.  Therefore:

* PINNED by in-tree reference code (checked by tests/test_oracle_golden.py against
  fixtures generated from the reference's own Python, tests/golden/make_golden.py):
    - SH basis / constants / +0.5 offset ....... utils/sh_utils.py:25-119
    - quaternion -> R, Sigma = (R S)(R S)^T, 6-float packing .. gs_renderer.py:79-92,124-157,168-172
    - camera matrix conventions (row-vector, w_clip = z_view) .. utils/graphics_utils.py:47-81,
      utils/cam_utils.py:182-210
    - output contract (color, radii, depth_alpha[2,H,W]; depth_alpha[1] = transmittance)
      .......................................... scene_gaussian.py:637-671,861-893
* PARITY UNPINNED (restated from the published 3DGS algorithm lineage, SURVEY.md App. A):
  0.2 near cull, 1.3*tanfov EWA clamp, +0.3 dilation, 3-sigma radius, 16x16 tiles,
  (tile<<32 | depth bits) key, alpha=min(0.99,.), 1/255 skip, T<1e-4 stop, the
  important_score definition (sum of blend weights alpha*T), every backward formula.

Numerics contract shared with the CUDA kernels (dreamscene_b200/csrc/project.cu)
-------------------------------------------------------------------------------
Everything that decides an INTEGER (depth bits, radius, tile rect, hence the sorted
tile lists) is evaluated in fp32 with every multiply/add individually rounded, no FMA
contraction, in exactly the order written in ``preprocess`` below.  The CUDA side uses
__fmul_rn/__fadd_rn/__fdiv_rn/__fsqrt_rn in the same order, so these integers are
bit-exact by construction.  Colours, conics and blending are float-tolerance quantities.

Autograd of this forward equals the analytic CUDA backward because the places where
the CUDA backward ignores a non-linearity are neutralised explicitly (SURVEY.md A.9):
straight-through 0.99 clamp, boolean skip/stop masks, EWA clamp treated as a constant.
"""
from __future__ import annotations

from dataclasses import dataclass
from typing import Optional

import numpy as np
import torch

BLOCK = 16
NEAR_Z = 0.2
ALPHA_MIN = 1.0 / 255.0
ALPHA_MAX = 0.99
T_STOP = 1e-4
DILATION = 0.3

# utils/sh_utils.py:25-53
SH_C0 = 0.28209479177387814
SH_C1 = 0.4886025119029199
SH_C2 = [1.0925484305920792, -1.0925484305920792, 0.31539156525252005,
         -1.0925484305920792, 0.5462742152960396]
SH_C3 = [-0.5900435899266435, 2.890611442640554, -0.4570457994644658,
         0.3731763325901154, -0.4570457994644658, 1.445305721320277,
         -0.5900435899266435]


@dataclass
class Settings:
    """Mirror of GaussianRasterizationSettings (scene_gaussian.py:586-599)."""
    image_height: int
    image_width: int
    tanfovx: float
    tanfovy: float
    bg: torch.Tensor
    scale_modifier: float
    viewmatrix: torch.Tensor
    projmatrix: torch.Tensor
    sh_degree: int
    campos: torch.Tensor
    prefiltered: bool = False
    score_flag: bool = False


def _c(v, dtype):
    return torch.tensor(float(v), dtype=dtype)


def eval_sh_basis_dot(deg: int, sh: torch.Tensor, d: torch.Tensor) -> torch.Tensor:
    """sh [P,M,3], d [P,3] unit dirs -> [P,3].  Follows utils/sh_utils.py:56-102 (deg<=3)."""
    res = SH_C0 * sh[:, 0]
    if deg > 0:
        x, y, z = d[:, 0:1], d[:, 1:2], d[:, 2:3]
        res = res - SH_C1 * y * sh[:, 1] + SH_C1 * z * sh[:, 2] - SH_C1 * x * sh[:, 3]
        if deg > 1:
            xx, yy, zz = x * x, y * y, z * z
            xy, yz, xz = x * y, y * z, x * z
            res = (res + SH_C2[0] * xy * sh[:, 4] + SH_C2[1] * yz * sh[:, 5]
                   + SH_C2[2] * (2.0 * zz - xx - yy) * sh[:, 6]
                   + SH_C2[3] * xz * sh[:, 7] + SH_C2[4] * (xx - yy) * sh[:, 8])
            if deg > 2:
                res = (res + SH_C3[0] * y * (3 * xx - yy) * sh[:, 9]
                       + SH_C3[1] * xy * z * sh[:, 10]
                       + SH_C3[2] * y * (4 * zz - xx - yy) * sh[:, 11]
                       + SH_C3[3] * z * (2 * zz - 3 * xx - 3 * yy) * sh[:, 12]
                       + SH_C3[4] * x * (4 * zz - xx - yy) * sh[:, 13]
                       + SH_C3[5] * z * (xx - yy) * sh[:, 14]
                       + SH_C3[6] * x * (xx - 3 * yy) * sh[:, 15])
    return res


def cov3d_from_scale_rot(scales: torch.Tensor, rots: torch.Tensor, scale_modifier, dtype):
    """Sigma = R S S^T R^T, packed (xx,xy,xz,yy,yz,zz).  gs_renderer.py:124-157,79-92.
    The quaternion is used AS GIVEN (the caller normalises: gs_renderer.py:469-470)."""
    mod = _c(scale_modifier, dtype)
    s0, s1, s2 = mod * scales[:, 0], mod * scales[:, 1], mod * scales[:, 2]
    r, x, y, z = rots[:, 0], rots[:, 1], rots[:, 2], rots[:, 3]
    R = [[1 - 2 * (y * y + z * z), 2 * (x * y - r * z), 2 * (x * z + r * y)],
         [2 * (x * y + r * z), 1 - 2 * (x * x + z * z), 2 * (y * z - r * x)],
         [2 * (x * z - r * y), 2 * (y * z + r * x), 1 - 2 * (x * x + y * y)]]
    L = [[R[i][0] * s0, R[i][1] * s1, R[i][2] * s2] for i in range(3)]

    def dot(i, j):
        return (L[i][0] * L[j][0] + L[i][1] * L[j][1]) + L[i][2] * L[j][2]

    return torch.stack([dot(0, 0), dot(0, 1), dot(0, 2), dot(1, 1), dot(1, 2), dot(2, 2)], dim=1)


def preprocess(S: Settings, means3D, opacities, shs=None, colors_precomp=None, scales=None,
               rotations=None, cov3D_precomp=None, means2D=None, dtype=torch.float32,
               decisions: Optional[dict] = None):
    """Per-Gaussian stage (SURVEY.md A.1-A.5).  Differentiable.  Returns a dict.

    ``decisions``: integer decisions (visible/radii/rect) from another run (used to evaluate
    the fp64 gradient reference on exactly the fp32 pair lists).  When they also hold the branch
    flags ``in_x`` / ``in_y`` (EWA clamp) and ``clamped`` (SH colour clamp), those are used in
    place of the flags this run would compute in its own dtype: a Gaussian whose t.x/t.z lies
    within an ulp of the clamp limit, or whose colour lies within an ulp of 0, would otherwise take
    the other gradient branch in fp64 (identity vs zero) than in the fp32 run it is compared with."""
    P = means3D.shape[0]
    H, W = int(S.image_height), int(S.image_width)
    V = S.viewmatrix.detach().to("cpu", dtype).reshape(16)
    F = S.projmatrix.detach().to("cpu", dtype).reshape(16)
    campos = S.campos.detach().to("cpu", dtype).reshape(3)
    x, y, z = means3D[:, 0], means3D[:, 1], means3D[:, 2]

    # A.1 view / clip transforms (row-vector convention: flat index 4*r + c)
    tx = ((V[0] * x + V[4] * y) + V[8] * z) + V[12]
    ty = ((V[1] * x + V[5] * y) + V[9] * z) + V[13]
    tz = ((V[2] * x + V[6] * y) + V[10] * z) + V[14]
    hx = ((F[0] * x + F[4] * y) + F[8] * z) + F[12]
    hy = ((F[1] * x + F[5] * y) + F[9] * z) + F[13]
    hw = ((F[3] * x + F[7] * y) + F[11] * z) + F[15]
    pw = 1.0 / (hw + _c(1e-7, dtype))
    ndcx, ndcy = hx * pw, hy * pw
    if means2D is not None:  # gradient-only port, NDC units (A.9)
        ndcx = ndcx + means2D[:, 0]
        ndcy = ndcy + means2D[:, 1]
    Wf, Hf = _c(W, dtype), _c(H, dtype)
    px = ((ndcx + 1.0) * Wf - 1.0) * 0.5
    py = ((ndcy + 1.0) * Hf - 1.0) * 0.5

    # A.2 covariance
    if cov3D_precomp is not None:
        cov3D = cov3D_precomp
    else:
        cov3D = cov3d_from_scale_rot(scales, rotations, S.scale_modifier, dtype)
    c_xx, c_xy, c_xz, c_yy, c_yz, c_zz = [cov3D[:, i] for i in range(6)]
    Sg = [[c_xx, c_xy, c_xz], [c_xy, c_yy, c_yz], [c_xz, c_yz, c_zz]]

    # A.3 EWA projection
    tfx, tfy = _c(S.tanfovx, dtype), _c(S.tanfovy, dtype)
    limx, limy = _c(1.3, dtype) * tfx, _c(1.3, dtype) * tfy
    fx, fy = Wf / (_c(2.0, dtype) * tfx), Hf / (_c(2.0, dtype) * tfy)
    with torch.no_grad():
        tz_safe = torch.where(tz == 0, torch.ones_like(tz), tz)
        txtz, tytz = tx / tz_safe, ty / tz_safe
        if decisions is not None and "in_x" in decisions:
            in_x, in_y = decisions["in_x"], decisions["in_y"]
        else:
            in_x = (txtz >= -limx) & (txtz <= limx)
            in_y = (tytz >= -limy) & (tytz <= limy)
        cx_val = torch.minimum(limx, torch.maximum(-limx, txtz)) * tz
        cy_val = torch.minimum(limy, torch.maximum(-limy, tytz)) * tz
    # value = clamp(t.x/t.z)*t.z ; gradient = identity when unclamped, constant when clamped
    cx = cx_val + torch.where(in_x, tx - tx.detach(), torch.zeros_like(tx))
    cy = cy_val + torch.where(in_y, ty - ty.detach(), torch.zeros_like(ty))
    # (culled Gaussians never reach the outputs; tz==0 only occurs among them)
    tzd = torch.where(tz.detach() == 0, torch.ones_like(tz), tz)
    J00 = fx / tzd
    J02 = -(fx * cx) / (tzd * tzd)
    J11 = fy / tzd
    J12 = -(fy * cy) / (tzd * tzd)
    Wr = [[V[4 * k + i] for k in range(3)] for i in range(3)]  # Wr[i][k] = V[k][i]
    M0 = [J00 * Wr[0][k] + J02 * Wr[2][k] for k in range(3)]
    M1 = [J11 * Wr[1][k] + J12 * Wr[2][k] for k in range(3)]
    N0 = [(M0[0] * Sg[0][j] + M0[1] * Sg[1][j]) + M0[2] * Sg[2][j] for j in range(3)]
    N1 = [(M1[0] * Sg[0][j] + M1[1] * Sg[1][j]) + M1[2] * Sg[2][j] for j in range(3)]
    a = ((N0[0] * M0[0] + N0[1] * M0[1]) + N0[2] * M0[2]) + _c(DILATION, dtype)
    b = (N0[0] * M1[0] + N0[1] * M1[1]) + N0[2] * M1[2]
    c = ((N1[0] * M1[0] + N1[1] * M1[1]) + N1[2] * M1[2]) + _c(DILATION, dtype)
    det = a * c - b * b
    det_safe = torch.where(det.detach() == 0, torch.ones_like(det), det)
    det_inv = 1.0 / det_safe
    con_a, con_b, con_c = c * det_inv, -b * det_inv, a * det_inv

    gx, gy = (W + BLOCK - 1) // BLOCK, (H + BLOCK - 1) // BLOCK
    if decisions is None:
        with torch.no_grad():
            mid = 0.5 * (a + c)
            sq = torch.sqrt(torch.clamp_min(mid * mid - det, 0.1))
            lam = torch.maximum(mid + sq, mid - sq)
            rad_f = torch.ceil(3.0 * torch.sqrt(lam))
            rad_f = torch.nan_to_num(rad_f, nan=0.0, posinf=1.0e9, neginf=0.0).clamp(0.0, 1.0e9)
            radius = rad_f.to(torch.int64)
            front = tz > _c(NEAR_Z, dtype)
            ok = front & (det != 0)

            def tile(v, g):
                t = torch.nan_to_num(v / BLOCK, nan=0.0).clamp(-1.0, float(g) + 1.0)
                return torch.trunc(t).to(torch.int64).clamp(0, g)

            rminx, rmaxx = tile(px - rad_f, gx), tile(px + rad_f + (BLOCK - 1), gx)
            rminy, rmaxy = tile(py - rad_f, gy), tile(py + rad_f + (BLOCK - 1), gy)
            touched = (rmaxx - rminx) * (rmaxy - rminy)
            visible = ok & (touched > 0)
            touched = torch.where(visible, touched, torch.zeros_like(touched))
            radii = torch.where(visible, radius, torch.zeros_like(radius)).to(torch.int32)
            rect = torch.stack([rminx, rminy, rmaxx, rmaxy], dim=1)
    else:
        visible, radii, rect, touched = (decisions[k] for k in ("visible", "radii", "rect", "touched"))

    # A.5 colour
    clamped = None
    if shs is not None:
        d = means3D - campos[None, :]
        dn = torch.sqrt((d[:, 0] * d[:, 0] + d[:, 1] * d[:, 1]) + d[:, 2] * d[:, 2])
        dn = torch.where(dn.detach() == 0, torch.ones_like(dn), dn)
        d = d / dn[:, None]
        raw = eval_sh_basis_dot(int(S.sh_degree), shs, d) + 0.5
        if decisions is not None and decisions.get("clamped") is not None:
            clamped = decisions["clamped"]
        else:
            clamped = (raw.detach() < 0)
        # = clamp_min(raw, 0) in value and gradient when `clamped` is this run's own mask
        rgb = torch.where(clamped, torch.zeros_like(raw), raw)
    else:
        rgb = colors_precomp

    return dict(depth=tz, px=px, py=py, conic=(con_a, con_b, con_c), opacity=opacities.reshape(P),
                rgb=rgb, cov2d=(a, b, c), cov3D=cov3D, radii=radii, rect=rect, touched=touched,
                visible=visible, in_x=in_x, in_y=in_y, clamped=clamped, grid=(gx, gy))


def bin_and_sort(pre, S: Settings):
    """A.6 first half: emit (tile<<32 | depth_bits, idx), stable sort, per-tile ranges.
    depth bits are the fp32 bits of pre['depth'] (must come from an fp32 run)."""
    gx, gy = pre["grid"]
    vis = pre["visible"].numpy()
    rect = pre["rect"].numpy()
    touched = pre["touched"].numpy().astype(np.int64)
    depth32 = pre["depth"].detach().to(torch.float32).numpy()
    idx = np.nonzero(vis)[0]
    cnt = touched[idx]
    D = int(cnt.sum())
    if D == 0:
        return (np.zeros(0, np.uint64), np.zeros(0, np.int64),
                np.zeros((gx * gy, 2), np.int64))
    rep = np.repeat(idx, cnt)
    start = np.cumsum(cnt) - cnt
    local = np.arange(D, dtype=np.int64) - np.repeat(start, cnt)
    w = (rect[rep, 2] - rect[rep, 0]).astype(np.int64)
    ly, lx = local // w, local % w
    tile = (rect[rep, 1] + ly) * gx + (rect[rep, 0] + lx)
    keys = (tile.astype(np.uint64) << np.uint64(32)) | depth32.view(np.uint32)[rep].astype(np.uint64)
    order = np.argsort(keys, kind="stable")
    keys_s, point_list = keys[order], rep[order]
    tile_s = (keys_s >> np.uint64(32)).astype(np.int64)
    ntiles = gx * gy
    starts = np.searchsorted(tile_s, np.arange(ntiles), side="left")
    ends = np.searchsorted(tile_s, np.arange(ntiles), side="right")
    return keys_s, point_list.astype(np.int64), np.stack([starts, ends], axis=1).astype(np.int64)


def composite(pre, point_list, ranges, S: Settings, dtype=torch.float32, tiles=None,
              max_chunk=4096, record_blend: Optional[dict] = None, replay_blend: Optional[dict] = None):
    """A.6 second half.  Differentiable front-to-back blend, one tile at a time.

    Returns color[3,H,W], depth_alpha[2,H,W], n_contrib[H,W] (int32), score[P] (or None).

    record_blend / replay_blend: the per-(entry, pixel) blend decisions (alpha >= 1/255, power <= 0,
    T stop) are discontinuous, so an fp64 evaluation flips a handful of borderline pairs relative to
    fp32 and a single flipped pair dominates a norm-wise gradient comparison.  An fp32 run can record
    its decisions ({(tile, chunk start): (blend mask, stopped-at-end mask)}) and an fp64 run replay
    them: the fp64 gradient is then evaluated on exactly the fp32 decision set."""
    H, W = int(S.image_height), int(S.image_width)
    gx, gy = pre["grid"]
    bg = S.bg.detach().to("cpu", dtype).reshape(3)
    P = pre["px"].shape[0]
    color = torch.zeros(3, H, W, dtype=dtype) + bg[:, None, None]
    dacc = torch.zeros(H, W, dtype=dtype)
    tfin = torch.ones(H, W, dtype=dtype)
    ncon = torch.zeros(H, W, dtype=torch.int32)
    score = torch.zeros(P, dtype=dtype) if S.score_flag else None
    con_a, con_b, con_c = pre["conic"]
    pl = torch.from_numpy(np.ascontiguousarray(point_list))
    amin, amax, tstop = _c(ALPHA_MIN, dtype), _c(ALPHA_MAX, dtype), _c(T_STOP, dtype)
    col_out, d_out, t_out = [], [], []
    tile_ids = range(gx * gy) if tiles is None else tiles
    for t in tile_ids:
        s, e = int(ranges[t, 0]), int(ranges[t, 1])
        if e <= s:
            continue
        ty_, tx_ = divmod(t, gx)
        x0, y0 = tx_ * BLOCK, ty_ * BLOCK
        x1, y1 = min(x0 + BLOCK, W), min(y0 + BLOCK, H)
        ys, xs = torch.meshgrid(torch.arange(y0, y1), torch.arange(x0, x1), indexing="ij")
        X = xs.reshape(1, -1).to(dtype)
        Y = ys.reshape(1, -1).to(dtype)
        npix = X.shape[1]
        T_run = torch.ones(npix, dtype=dtype)
        C_run = torch.zeros(npix, 3, dtype=dtype)
        D_run = torch.zeros(npix, dtype=dtype)
        last = torch.zeros(npix, dtype=torch.int64)
        alive = torch.ones(npix, dtype=torch.bool)
        for cs in range(s, e, max_chunk):
            ce = min(e, cs + max_chunk)
            ids = pl[cs:ce]
            dx = pre["px"][ids][:, None] - X
            dy = pre["py"][ids][:, None] - Y
            A_, B_, C_ = con_a[ids][:, None], con_b[ids][:, None], con_c[ids][:, None]
            power = -0.5 * (A_ * dx * dx + C_ * dy * dy) - B_ * dx * dy
            G = torch.exp(torch.clamp_max(power, 0.0))
            araw = pre["opacity"][ids][:, None] * G
            alpha = araw + (torch.clamp_max(araw, amax) - araw).detach()
            with torch.no_grad():
                if replay_blend is not None:
                    blend, stopped_end = replay_blend[(t, cs)]
                else:
                    valid = (power <= 0) & (alpha >= amin) & alive[None, :]
                    om = torch.where(valid, 1.0 - alpha, torch.ones_like(alpha))
                    T_incl = torch.cumprod(om, dim=0) * T_run.detach()[None, :]
                    stop = valid & (T_incl < tstop)
                    stopped = torch.cumsum(stop.to(torch.int32), dim=0) > 0
                    blend = valid & ~stopped
                    stopped_end = stopped[-1]
                    if record_blend is not None:
                        record_blend[(t, cs)] = (blend.clone(), stopped_end.clone())
            omb = torch.where(blend, 1.0 - alpha, torch.ones_like(alpha))
            T_in = torch.cumprod(omb, dim=0)
            T_before = torch.cat([torch.ones(1, npix, dtype=dtype), T_in[:-1]], dim=0) * T_run[None, :]
            wgt = torch.where(blend, alpha * T_before, torch.zeros_like(alpha))
            C_run = C_run + torch.einsum("np,nc->pc", wgt, pre["rgb"][ids])
            D_run = D_run + (wgt * pre["depth"][ids][:, None]).sum(0)
            T_run = T_run * T_in[-1]
            with torch.no_grad():
                pos = torch.arange(cs - s + 1, ce - s + 1)[:, None]
                last = torch.maximum(last, (blend * pos).max(dim=0).values)
                alive = alive & ~stopped_end
                if score is not None:
                    score.index_add_(0, ids, wgt.sum(1))
            if not bool(alive.any()):
                break
        col = C_run.t() + T_run[None, :] * bg[:, None]
        col_out.append((col, D_run, T_run, last, (ys.reshape(-1) * W + xs.reshape(-1))))
    # scatter tiles into images with ONE differentiable index_copy per channel group
    if col_out:
        pix = torch.cat([c[4] for c in col_out])
        color = torch.index_copy(color.reshape(3, H * W), 1, pix,
                                 torch.cat([c[0] for c in col_out], dim=1)).reshape(3, H, W)
        dacc = torch.index_copy(dacc.reshape(H * W), 0, pix,
                                torch.cat([c[1] for c in col_out])).reshape(H, W)
        tfin = torch.index_copy(tfin.reshape(H * W), 0, pix,
                                torch.cat([c[2] for c in col_out])).reshape(H, W)
        ncon = torch.index_copy(ncon.reshape(H * W), 0, pix,
                                torch.cat([c[3] for c in col_out]).to(torch.int32)).reshape(H, W)
    return color, torch.stack([dacc, tfin], dim=0), ncon, score


def rasterize(S: Settings, means3D, opacities, shs=None, colors_precomp=None, scales=None,
              rotations=None, cov3D_precomp=None, means2D=None, dtype=torch.float32,
              decisions: Optional[dict] = None, tiles=None, record_blend: Optional[dict] = None):
    """Full forward.  Returns dict(color, depth_alpha, radii, score, + intermediates).

    ``decisions`` (optional) = {'visible','radii','rect','touched','point_list','ranges'} from a
    previous fp32 run; lets an fp64 run use the bit-exact fp32 pair lists.  The decisions this
    returns also carry the branch flags 'in_x', 'in_y' and 'clamped' (see ``preprocess``), so an
    fp64 run given them takes the fp32 run's gradient branch on every Gaussian."""
    if (shs is None) == (colors_precomp is None):
        raise Exception("Please provide excatly one of either SHs or precomputed colors!")
    if ((scales is None or rotations is None) and cov3D_precomp is None) or \
       ((scales is not None or rotations is not None) and cov3D_precomp is not None):
        raise Exception("Please provide exactly one of either scale/rotation pair or precomputed 3D covariance!")
    cast = lambda t: None if t is None else t.to(dtype)
    pre = preprocess(S, cast(means3D), cast(opacities), cast(shs), cast(colors_precomp),
                     cast(scales), cast(rotations), cast(cov3D_precomp), cast(means2D), dtype,
                     decisions)
    if decisions is not None and "point_list" in decisions:
        keys, point_list, ranges = None, decisions["point_list"], decisions["ranges"]
    else:
        keys, point_list, ranges = bin_and_sort(pre, S)
    replay = decisions.get("blend") if decisions is not None else None
    color, depth_alpha, ncon, score = composite(pre, point_list, ranges, S, dtype, tiles,
                                                record_blend=record_blend, replay_blend=replay)
    return dict(color=color, depth_alpha=depth_alpha, radii=pre["radii"], score=score,
                n_contrib=ncon, keys=keys, point_list=point_list, ranges=ranges, pre=pre,
                decisions=dict(visible=pre["visible"], radii=pre["radii"], rect=pre["rect"],
                               touched=pre["touched"], point_list=point_list, ranges=ranges,
                               in_x=pre["in_x"], in_y=pre["in_y"], clamped=pre["clamped"],
                               **({"blend": record_blend} if record_blend is not None else {})))
