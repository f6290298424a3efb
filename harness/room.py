"""The indoor scene of BASELINE.json config 5 (cfg5): a 6 x 5 x 2.8 m room (four walls, a ceiling and a floor) with
four ball-shaped objects inside, built with the reference's init recipes (gs_renderer.py:218-248 walls, 279-296
floor; configs/scenes/sample_indoor.yaml box), and the cameras inside it that DreamScene's scene stages render
from.  benchmarks/scene_step.py and the benchmarks built on it render this scene; tests/test_gpu_room.py checks the
rasterizer against the oracle on it (harness code: the product never imports it).

build_scene(dev) with the default sizes is cfg5 (2.63 M Gaussians); n_wall / n_floor / n_obj shrink it to a room the
CPU oracle can render in full, and scale_mul widens its Gaussians so that the smaller room is about as opaque."""
import math

import numpy as np
import torch

from harness import cameras
from harness.scene_ref import reference_assemble

SH_C0 = 0.28209479177387814
ROOM = (6.0, 5.0, 2.8)                 # room box (m): x, y, z; the floor is z = 0, the centre of the floor x = y = 0
OBJECT_CENTRES = ([1.0, 0.8, 0.5], [-1.2, -0.6, 0.4], [0.3, -1.3, 0.45], [-0.5, 1.2, 0.6])


def plane_points(n, origin, u, v, rng):
    a, b = rng.random_sample((n, 1)), rng.random_sample((n, 1))
    return origin[None] + a * u[None] + b * v[None]


def make_group(xyz, rng, M, dev, scale):
    P = xyz.shape[0]
    t = lambda a: torch.tensor(np.ascontiguousarray(a, dtype=np.float32), device=dev)
    return dict(
        xyz=t(xyz).requires_grad_(True),
        f_dc=t((rng.random_sample((P, 1, 3)) - 0.5) / SH_C0).requires_grad_(True),
        f_rest=t(rng.normal(0, 0.02, (P, M - 1, 3))).requires_grad_(True),
        scaling=t(np.log(np.full((P, 3), scale) * np.exp(rng.normal(0, 0.2, (P, 3))))).requires_grad_(True),
        rotation=t(np.tile([1.0, 0, 0, 0], (P, 1)) + rng.normal(0, 0.05, (P, 4))).requires_grad_(True),
        opacity=t(np.full((P, 1), math.log(0.1 / 0.9))).requires_grad_(True))


def build_scene(dev, M=4, n_wall=400_000, n_floor=300_000, n_obj=81_920, seed=0, scale_mul=1.0):
    """-> [env (4 walls + ceiling), floor, 4 objects]: groups of raw leaves (xyz, f_dc, f_rest, scaling, rotation,
    opacity) as GaussianModel holds them.  n_wall Gaussians per wall and on the ceiling, n_floor on the floor, n_obj
    per object; scale_mul multiplies every Gaussian's scale."""
    rng = np.random.RandomState(seed)
    L, Wd, Hh = ROOM
    o = np.array([-L / 2, -Wd / 2, 0.0])
    ex, ey, ez = np.array([L, 0, 0.0]), np.array([0, Wd, 0.0]), np.array([0, 0, Hh])
    walls = [plane_points(n_wall, o, ex, ez, rng), plane_points(n_wall, o + ey, ex, ez, rng),
             plane_points(n_wall, o, ey, ez, rng), plane_points(n_wall, o + ex, ey, ez, rng),
             plane_points(n_wall, o + ez, ex, ey, rng)]                     # 4 walls + ceiling
    env = make_group(np.concatenate(walls), rng, M, dev, scale=0.008 * scale_mul)
    floor = make_group(plane_points(n_floor, o, ex, ey, rng), rng, M, dev, scale=0.008 * scale_mul)
    objs = []
    for c in OBJECT_CENTRES:
        d = rng.normal(size=(n_obj, 3)); d /= np.linalg.norm(d, axis=1, keepdims=True)
        xyz = np.array(c)[None] + 0.35 * np.cbrt(rng.random_sample((n_obj, 1))) * d
        objs.append(make_group(xyz, rng, M, dev, scale=0.006 * scale_mul))
    return [env, floor] + objs


def look_camera(eye, fwd, size, dev, fovx=0.96):
    """Camera at `eye` looking along the unit vector `fwd`, the world's +z up (cameras.orbit_pose's axes)."""
    fwd = np.asarray(fwd, np.float32)
    up = np.array([0, 0, 1], np.float32)
    right = np.cross(fwd, up); right /= np.linalg.norm(right)
    up = np.cross(right, fwd)
    pose = np.eye(4, dtype=np.float32)
    pose[:3, :3] = np.stack((-right, up, -fwd), axis=-1)
    pose[:3, 3] = np.asarray(eye, np.float32)
    return cameras.camera_from_pose(pose, fovx, size, size, device=dev)


def scene_camera(k, size, dev):
    # camera inside the room, looking roughly horizontally (Stage1_Indoor-like), FoV 0.96
    ang = 2 * math.pi * (k * 0.37 % 1.0)
    eye = np.array([0.8 * math.cos(ang * 1.7), 0.6 * math.sin(ang * 1.3), 1.4], np.float32)
    fwd = np.array([math.cos(ang), math.sin(ang), -0.1], np.float32); fwd /= np.linalg.norm(fwd)
    return look_camera(eye, fwd, size, dev, 0.96)


def named_groups(groups):
    """The groups under GaussianModel's attribute names, as assemble_scene / render_scene take them."""
    return [{"_xyz": g["xyz"], "_opacity": g["opacity"], "_scaling": g["scaling"], "_rotation": g["rotation"],
             "_features_dc": g["f_dc"], "_features_rest": g["f_rest"]} for g in groups]


def rasterizer_inputs(groups):
    """The activated rasterizer inputs of the whole scene without augmentation (reference_assemble), detached, as
    CPU tensors in the oracle's names: dict(means3D, opacities, shs, scales, rotations)."""
    with torch.no_grad():
        xyz, opacity, scales, rots, shs = reference_assemble(named_groups(groups))
    return {k: v.detach().cpu().contiguous() for k, v in
            (("means3D", xyz), ("opacities", opacity), ("shs", shs), ("scales", scales), ("rotations", rots))}
