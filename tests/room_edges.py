"""Gaussians built on the rasterizer's branch boundaries, for an axis-aligned camera whose view matrix holds only
exact 0 / +-1 entries and no translation along its view x and z axes: t.z and t.x are then the world coordinates
themselves, bit for bit, so the near plane and the EWA clamp limit can be hit exactly and one fp32 ulp either side.
Every constructed value is re-derived through the oracle's fp32 operation chain rather than assumed.

Shared by the CPU replay test of the oracle (test_oracle_properties.py) and the room tests on the GPU."""
import math

import numpy as np
import torch

from harness import room
from oracle import splat_ref as O

f32 = np.float32
AXIS_EYE = (0.0, 0.0, 1.4)          # on the room's centre line, looking along +x


def axis_camera(size, dev="cpu"):
    return room.look_camera(AXIS_EYE, [1.0, 0.0, 0.0], size, dev)


def view_f32(V, pts):
    """fp32 view-space (tx, ty, tz) of world points [n,3], the oracle's operation order."""
    V = np.asarray(V, np.float32).reshape(16)
    x, y, z = (np.asarray(pts, np.float32)[:, k] for k in range(3))
    tx = ((V[0] * x + V[4] * y) + V[8] * z) + V[12]
    ty = ((V[1] * x + V[5] * y) + V[9] * z) + V[13]
    tz = ((V[2] * x + V[6] * y) + V[10] * z) + V[14]
    return tx, ty, tz


def check_axis_camera(cam):
    """The camera the constructions rely on: rotation entries exactly 0 / +-1, t.x = y and t.z = x exactly."""
    V = cam.world_view_transform.numpy().astype(np.float32)
    assert set(np.abs(V[:3, :3]).ravel().tolist()) <= {0.0, 1.0}
    assert V[3, 0] == 0.0 and V[3, 2] == 0.0 and V[3, 3] == 1.0
    assert V[1, 0] == 1.0 and V[0, 2] == 1.0                   # t.x = +y, t.z = +x
    return V


def limits(cam):
    """fp32 EWA clamp limits (1.3 * tanfov), as project.cu / the oracle compute them."""
    return f32(1.3) * f32(cam.tanfovx), f32(1.3) * f32(cam.tanfovy)


def _ulps(v, k):
    v = f32(v)
    for _ in range(abs(k)):
        v = np.nextafter(v, f32(np.inf) if k > 0 else f32(-np.inf))
    return f32(v)


def point_at_ratio(cam, axis, target, tz0, other, K=96):
    """A world point whose fp32 t.{axis}/t.z equals `target` bit for bit, t.z near tz0 and the other view-plane
    coordinate near `other`.  Searches the fp32 neighbourhood (the y translation of the camera makes t.y coarser
    than t.y/t.z, so a direct construction does not exist for every target)."""
    V = check_axis_camera(cam)
    xs = np.array([_ulps(tz0, k) for k in range(-K, K + 1)], np.float32)          # world x = t.z
    if axis == "x":
        ws = np.array([_ulps(target * tz0, k) for k in range(-K, K + 1)], np.float32)  # world y = t.x
        pts = np.stack(np.broadcast_arrays(xs[:, None], ws[None, :], f32(AXIS_EYE[2] - other)), -1).reshape(-1, 3)
    else:
        z0 = f32(AXIS_EYE[2] - target * tz0)                                          # t.y = 1.4 - z
        ws = np.array([_ulps(z0, k) for k in range(-K, K + 1)], np.float32)
        pts = np.stack(np.broadcast_arrays(xs[:, None], f32(other), ws[None, :]), -1).reshape(-1, 3)
    tx, ty, tz = view_f32(V, pts)
    q = (tx if axis == "x" else ty) / tz
    hit = np.nonzero(q == f32(target))[0]
    assert hit.size, f"no fp32 point with t.{axis}/t.z == {target!r} near t.z = {tz0}"
    return pts[hit[0]].astype(np.float32)


def zero_colour_dc(k):
    """An SH DC coefficient (the other coefficients 0) whose fp32 colour  SH_C0 * dc + 0.5  is exactly 0 (k = 0) or
    k fp32 ulps of dc away from it."""
    c0 = f32(O.SH_C0)
    dc = f32(-0.5) / c0
    for _ in range(64):                       # the dc nearest to -0.5 / C0 whose product rounds to exactly -0.5
        if f32(c0 * dc) == f32(-0.5):
            break
        dc = np.nextafter(dc, f32(np.inf) if f32(c0 * dc) < f32(-0.5) else f32(-np.inf))
    assert f32(c0 * dc) + f32(0.5) == f32(0.0)
    return _ulps(dc, k)


def _row(mean, scale, quat=(1.0, 0.0, 0.0, 0.0), opacity=0.5, dc=None, rng=None, kind="", rest=None):
    dc = rng.uniform(-1.0, 1.0, 3) if dc is None else np.full(3, dc)
    return dict(mean=np.asarray(mean, np.float32), scale=np.asarray(scale, np.float32),
                quat=np.asarray(quat, np.float32), opacity=f32(opacity), dc=dc.astype(np.float32), kind=kind,
                rest=rest)


def colour_flip_row(cam, rng, mean=(1.5, 0.2, 1.3)):
    """A row whose colour the oracle clamps in fp32 and not in fp64, or the other way round: the DC coefficient near
    the zero of the colour and a small degree-1 coefficient (finer control than the DC ulps alone), searched."""
    S = O.Settings(cam.image_height, cam.image_width, cam.tanfovx, cam.tanfovy, torch.ones(3), 1.0,
                   cam.world_view_transform, cam.full_proj_transform, 1, cam.camera_center)
    # the degree-1 term moves the colour by less than an ulp of the DC product: t up to 2e-7
    cands = [(zero_colour_dc(k), f32(t)) for t in np.linspace(-2e-7, 2e-7, 81) for k in (-1, 0, 1)]
    n = len(cands)
    shs = np.zeros((n, 4, 3), np.float32)
    shs[:, 0] = np.array([c[0] for c in cands], np.float32)[:, None]
    shs[:, 3] = np.array([c[1] for c in cands], np.float32)[:, None]
    ins = dict(means3D=torch.from_numpy(np.tile(np.asarray(mean, np.float32), (n, 1))),
               opacities=torch.full((n, 1), 0.5), shs=torch.from_numpy(shs),
               scales=torch.full((n, 3), 0.05), rotations=torch.tensor([[1.0, 0.0, 0.0, 0.0]]).repeat(n, 1))
    flags = [O.preprocess(S, **{k: v.to(dt) for k, v in ins.items()}, dtype=dt)["clamped"][:, 0]
             for dt in (torch.float32, torch.float64)]
    hit = np.nonzero((flags[0] != flags[1]).numpy())[0]
    assert hit.size, "no colour near 0 whose fp32 and fp64 clamp decisions differ"
    dc, t = cands[int(hit[0])]
    rest = np.zeros((3, 3), np.float32)
    rest[2] = t                                        # coefficient 3 (the x term of degree 1)
    return _row(mean, [0.05] * 3, dc=dc, rng=rng, kind="colour_flip", rest=rest)


def boundary_rows(cam, rng, colour_flip=False):
    """Clamp-limit and colour-clamp boundaries: t.x/t.z and t.y/t.z = +-limit and one ulp either side, fp32 colours
    exactly 0 ("colour0_exact") and one ulp of the DC coefficient either side.  The kernels evaluate the colour with
    fused multiply-adds, so where the oracle's separately rounded fp32 gives exactly 0 they see -7e-9 and clamp
    (DESIGN.md section 8 item 8).  colour_flip: also a row whose fp32 and fp64 clamp decisions differ (colour_flip_row;
    the CPU replay test)."""
    limx, limy = limits(cam)
    rows = []
    for axis, lim in (("x", limx), ("y", limy)):
        for s in (1, -1):
            for d in (-1, 0, 1):
                p = point_at_ratio(cam, axis, _ulps(f32(s) * lim, d), f32(0.5), f32(0.03))
                rows.append(_row(p, [0.06] * 3, rng=rng, kind=f"ratio_{axis}"))
    for k in (-1, 0, 1):
        rows.append(_row([1.5, 0.1 * k, 1.3], [0.05] * 3, dc=zero_colour_dc(k), rng=rng,
                         kind="colour0_exact" if k == 0 else "colour0"))
    if colour_flip:
        rows.append(colour_flip_row(cam, rng))
    return rows


def edge_rows(cam, rng):
    """Every constructed edge case except the near-singular footprints (see near_singular_rows)."""
    rows = boundary_rows(cam, rng)
    tfx, tfy = cam.tanfovx, cam.tanfovy
    z_of = lambda ty: AXIS_EYE[2] - ty                       # world z of a view-space t.y
    near = f32(O.NEAR_Z)
    for k in (-2, -1, 0, 1, 2):                              # t.z = fp32(0.2) and +-1, +-2 ulps
        rows.append(_row([_ulps(near, k), 0.012 * k, z_of(0.01)], [0.004] * 3, opacity=0.3, rng=rng, kind="near"))
    # footprints containing the camera centre: in front of the near plane, between it and the camera, behind it
    for tz, op in ((0.25, 0.15), (0.1, 0.5), (-0.05, 0.5)):
        rows.append(_row([tz, 0.02, z_of(-0.01)], [0.4] * 3, opacity=op, rng=rng, kind="contains_eye"))
    # behind the camera, scaled so that their unculled footprint would cover the image
    for tz, s in ((-0.3, 1.5), (-1.0, 3.0), (-0.19, 0.8)):
        rows.append(_row([tz, 0.1, z_of(0.05)], [s] * 3, opacity=0.9, rng=rng, kind="behind"))
    # footprints clipped on each side and each corner of the image
    for ix in (-1, 0, 1):
        for iy in (-1, 0, 1):
            if ix or iy:
                rows.append(_row([1.0, 1.1 * ix * tfx, z_of(1.1 * iy * tfy)], [0.15] * 3, opacity=0.4, rng=rng,
                                 kind="clipped"))
    # centres far off-screen (|px| >> W): large ones reach into the image through the clamped footprint, small not
    for sx, sy, s in ((6, 0, 2.0), (-6, 0, 2.0), (0, 6, 2.0), (0, -6, 2.0), (5, 5, 2.5), (8, 0, 0.01)):
        rows.append(_row([1.0, sx * tfx, z_of(sy * tfy)], [s] * 3, opacity=0.3, rng=rng, kind="offscreen"))
    return rows


def near_singular_rows(cam, rng):
    """Large flat Gaussians seen edge-on at t.z ~ 0.25, their thin axis across the view ray at 45 degrees on screen:
    cov2D = (rank one) + 0.3 I, so det = a c - b^2 cancels most of its bits."""
    c, s = math.cos(math.pi / 8), math.sin(math.pi / 8)     # 45 degrees about the view axis (world x)
    rows = []
    for tz in (0.25, 0.27, 0.3):                             # on the view axis: exactly edge-on
        rows.append(_row([tz, 0.0, AXIS_EYE[2]], [0.03, 2e-4, 0.03], quat=(c, s, 0.0, 0.0),
                         opacity=0.3, rng=rng, kind="near_singular"))
    return rows


def as_inputs(rows, M):
    """Rows -> activated rasterizer inputs (CPU, fp32): SH DC from the row, the M - 1 higher coefficients from its
    `rest` (0 when None)."""
    P = len(rows)
    shs = np.zeros((P, M, 3), np.float32)
    shs[:, 0] = np.stack([r["dc"] for r in rows])
    for i, r in enumerate(rows):
        if r["rest"] is not None:
            shs[i, 1:1 + len(r["rest"])] = r["rest"]
    return dict(means3D=torch.from_numpy(np.stack([r["mean"] for r in rows])),
                opacities=torch.from_numpy(np.array([[r["opacity"]] for r in rows], np.float32)),
                shs=torch.from_numpy(shs),
                scales=torch.from_numpy(np.stack([r["scale"] for r in rows])),
                rotations=torch.from_numpy(np.stack([r["quat"] for r in rows])))


def append(sc, extra):
    return {k: torch.cat([sc[k], extra[k]]).contiguous() for k in sc}
