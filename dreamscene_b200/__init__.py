"""dreamscene_b200: H100-native (sm_90a) differentiable 3D-Gaussian rasterizer for DreamScene.

Public surface = the reference extension's surface (see dreamscene_b200.rasterizer); import it
either as ``dreamscene_b200`` or through the drop-in alias package ``diff_gaussian_rasterization``.
"""
from .rasterizer import (GaussianRasterizationSettings, GaussianRasterizer, PairCapacityOverflow,
                         flush_checks, last_pair_count, rasterize_gaussians, set_pair_count_mode,
                         set_workspace_capacity)
from . import parallel
from .optim import GaussianAdam
from .graph import StepGraph

__all__ = ["GaussianRasterizationSettings", "GaussianRasterizer", "rasterize_gaussians",
           "set_workspace_capacity", "set_pair_count_mode", "flush_checks", "last_pair_count",
           "PairCapacityOverflow", "parallel", "GaussianAdam", "StepGraph"]
