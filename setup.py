"""Optional packaging: `pip install --no-build-isolation -e .` makes `diff_gaussian_rasterization`,
`simple_knn` and `dreamscene_b200` importable system-wide (DreamScene's README installs the
upstream extensions the same way: /root/reference/README.md:50-51).  The CUDA library is compiled
in-tree for sm_90a by dreamscene_b200/_build.py (nvcc required)."""
import os
import sys

from setuptools import setup
from setuptools.command.build_py import build_py

HERE = os.path.dirname(os.path.abspath(__file__))


class BuildWithCuda(build_py):
    def run(self):
        sys.path.insert(0, HERE)
        from dreamscene_b200 import _build
        _build.build()
        super().run()


setup(
    name="b200gsr",
    version="0.1.0",
    description="H100-native differentiable 3D-Gaussian rasterizer (drop-in for DreamScene's diff_gaussian_rasterization)",
    packages=["dreamscene_b200", "diff_gaussian_rasterization", "simple_knn"],
    package_data={"dreamscene_b200": ["libb200gsr.so", "csrc/*", "../include/b200gsr.h", "../include/b200gsr_scene.h"]},
    cmdclass={"build_py": BuildWithCuda},
    python_requires=">=3.9",
)
