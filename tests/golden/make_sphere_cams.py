"""Generate tests/golden/ref_sphere_cams.npz FROM THE REFERENCE'S OWN PYTHON (needs a DreamScene checkout; the
tests only read the stored output): the random sphere cameras of 3D Gaussian filtering, i.e. loadSphereCam ->
GenerateSphereCameras -> sphere_poses (utils/cam_utils.py:1322-1366,1847-1866) with the object trainer's camera
options (config.py: default_radius 3.5, default_fovy 0.55, 512 x 512).  The reference hard-codes CUDA
allocations; this script redirects them to the CPU (no reference file is modified or copied).

    python tests/golden/make_sphere_cams.py <path to the DreamScene checkout>
"""
import os
import sys

import numpy as np
import torch

REF = sys.argv[1]
sys.path.insert(0, REF)

_zeros = torch.zeros


def _cpu_zeros(*a, **k):
    k.pop("device", None)
    return _zeros(*a, **k)


torch.zeros = _cpu_zeros
torch.Tensor.cuda = lambda self, *a, **k: self

from utils.cam_utils import GenerateSphereCameras, RCamera    # noqa: E402


class Opt:
    default_radius = 3.5
    default_fovy = 0.55
    image_w = 512
    image_h = 512
    SSAA = 1
    device = "cpu"


out = {}
for k, (seed, n) in enumerate([(0, 48), (1234, 5)]):
    torch.manual_seed(seed)                                    # sphere_poses draws torch.randn(n, 3)
    infos = GenerateSphereCameras(Opt, n)
    cams = [RCamera(R=c.R, T=c.T, FoVx=c.FovX, FoVy=c.FovY, delta_polar=0, delta_azimuth=0, delta_radius=0, opt=Opt)
            for c in infos]
    out[f"set{k}_args"] = np.array([seed, n, Opt.default_radius, Opt.default_fovy, Opt.image_h, Opt.image_w], np.float64)
    out[f"set{k}_view"] = np.stack([c.world_view_transform.numpy() for c in cams])
    out[f"set{k}_fullproj"] = np.stack([c.full_proj_transform.numpy() for c in cams])
    out[f"set{k}_center"] = np.stack([c.camera_center.numpy() for c in cams])
    out[f"set{k}_fov"] = np.array([[c.FoVx, c.FoVy] for c in cams], np.float64)
out["n_sets"] = np.array([2])

dst = os.path.join(os.path.dirname(os.path.abspath(__file__)), "ref_sphere_cams.npz")
np.savez_compressed(dst, **out)
print("wrote", dst, {k: v.shape for k, v in out.items()})
