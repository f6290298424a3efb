"""Camera construction with DreamScene's conventions (host-side helper for tests/bench).

Restates (does not import) the reference math so that harnesses can run on a box where
/root/reference does not exist:
  * look-at orbit pose ............ utils/cam_utils.py:277-309 (circle_poses)
  * pose -> (R, T) ................ utils/cam_utils.py:1383-1386
  * world->view, projection ....... utils/graphics_utils.py:47-81
  * row-vector (transposed) storage, full_proj = view @ proj, camera_center
    ................................ utils/cam_utils.py:196-210
Checked against fixtures produced by the reference code in tests/golden/make_golden.py.
"""
from __future__ import annotations

import math
from typing import NamedTuple

import numpy as np
import torch


class OrbitCamera(NamedTuple):
    image_height: int
    image_width: int
    FoVx: float
    FoVy: float
    tanfovx: float
    tanfovy: float
    world_view_transform: torch.Tensor  # [4,4] row-vector convention (translation in last row)
    full_proj_transform: torch.Tensor   # [4,4]
    camera_center: torch.Tensor         # [3]


def _normalize(v: np.ndarray) -> np.ndarray:
    return v / np.sqrt(np.maximum((v * v).sum(-1, keepdims=True), 1e-20))


def orbit_pose(radius: float, theta_deg: float, phi_deg: float) -> np.ndarray:
    """Camera-to-world pose looking at the origin (cam_utils.py:277-309)."""
    th, ph = np.float32(theta_deg / 180 * np.pi), np.float32(phi_deg / 180 * np.pi)
    r = np.float32(radius)
    c = np.array([r * np.sin(th) * np.sin(ph), r * np.sin(th) * np.cos(ph), r * np.cos(th)], np.float32)
    fwd = _normalize(c)
    up = np.array([0, 0, 1], np.float32)
    right = _normalize(np.cross(fwd, up))
    up = _normalize(np.cross(right, fwd))
    pose = np.eye(4, dtype=np.float32)
    pose[:3, :3] = np.stack((-right, up, fwd), axis=-1)
    pose[:3, 3] = c
    return pose


def fov2focal(fov, pixels):
    return pixels / (2 * math.tan(fov / 2))


def focal2fov(focal, pixels):
    return 2 * math.atan(pixels / (2 * focal))


def camera_from_pose(pose: np.ndarray, fovx: float, height: int, width: int,
                     znear: float = 0.01, zfar: float = 100.0, device="cpu") -> OrbitCamera:
    m = np.linalg.inv(pose)
    R = -np.transpose(m[:3, :3])
    R[:, 0] = -R[:, 0]
    T = -m[:3, 3]
    fovy = focal2fov(fov2focal(fovx, height), width)   # cam_utils.py:1387 (sic: h/w swapped upstream)
    Rt = np.zeros((4, 4))
    Rt[:3, :3] = R.transpose()
    Rt[:3, 3] = T
    Rt[3, 3] = 1.0
    Rt = np.float32(np.linalg.inv(np.linalg.inv(Rt)))  # getWorld2View2 with trans=0, scale=1
    wvt = torch.tensor(Rt).transpose(0, 1)
    thy, thx = math.tan(fovy / 2), math.tan(fovx / 2)
    top, right = thy * znear, thx * znear
    Pm = torch.zeros(4, 4)
    Pm[0, 0] = 2.0 * znear / (2 * right)
    Pm[1, 1] = 2.0 * znear / (2 * top)
    Pm[3, 2] = 1.0
    Pm[2, 2] = zfar / (zfar - znear)
    Pm[2, 3] = -(zfar * znear) / (zfar - znear)
    proj = Pm.transpose(0, 1)
    full = wvt.unsqueeze(0).bmm(proj.unsqueeze(0)).squeeze(0)
    center = wvt.inverse()[3, :3]
    return OrbitCamera(height, width, fovx, fovy, math.tan(fovx * 0.5), math.tan(fovy * 0.5),
                       wvt.contiguous().to(device), full.contiguous().to(device),
                       center.contiguous().to(device))


def orbit_camera(radius=3.5, theta_deg=60.0, phi_deg=0.0, fovx=0.55, height=512, width=512,
                 device="cpu") -> OrbitCamera:
    return camera_from_pose(orbit_pose(radius, theta_deg, phi_deg), fovx, height, width, device=device)


def _safe_normalize(x: torch.Tensor) -> torch.Tensor:
    return x / torch.sqrt(torch.clamp(torch.sum(x * x, -1, keepdim=True), min=1e-20))


def sphere_poses(n: int, radius: float = 3.5, generator=None) -> np.ndarray:
    """[n, 4, 4] camera-to-world poses on a sphere around the origin, looking at it (cam_utils.py:1322-1336):
    centres from torch.randn(n, 3) (drawn from `generator`, else the global CPU generator), the look-at of
    orbit_pose."""
    centers = torch.randn(n, 3, generator=generator)
    centers /= torch.norm(centers, dim=1).unsqueeze(1).repeat(1, 3)
    centers *= torch.tensor([radius], dtype=torch.float32)
    fwd = _safe_normalize(centers)
    up = torch.tensor([[0.0, 0.0, 1.0]]).repeat(n, 1)
    right = _safe_normalize(torch.cross(fwd, up, dim=-1))
    up = _safe_normalize(torch.cross(right, fwd, dim=-1))
    poses = torch.eye(4, dtype=torch.float).unsqueeze(0).repeat(n, 1, 1)
    poses[:, :3, :3] = torch.stack((-right, up, fwd), dim=-1)
    poses[:, :3, 3] = centers
    return poses.numpy()


def sphere_cameras(n: int, radius: float = 3.5, fovx: float = 0.55, H: int = 512, W: int = 512, generator=None,
                   device="cpu") -> list:
    """The random sphere cameras of 3D Gaussian filtering (loadSphereCam -> GenerateSphereCameras,
    cam_utils.py:1338-1366,1847-1866; the object trainer uses 48 of them at radius 3.5, FoV 0.55, 512 x 512)."""
    return [camera_from_pose(p, fovx, H, W, device=device) for p in sphere_poses(n, radius, generator)]
