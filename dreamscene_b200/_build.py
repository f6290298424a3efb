"""In-tree build of libb200gsr.so (sm_90a only) with nvcc.  No torch dependency in the library."""
from __future__ import annotations

import os
import shutil
import subprocess
import sys

HERE = os.path.dirname(os.path.abspath(__file__))
CSRC = os.path.join(HERE, "csrc")
LIB = os.path.join(HERE, "libb200gsr.so")
SOURCES = ["api.cu", "project.cu", "binning.cu", "composite.cu", "knn.cu", "assemble.cu", "postprocess.cu", "densify.cu", "optim.cu"]
HEADERS = [os.path.join(CSRC, "common.cuh"), os.path.join(CSRC, "scene_math.cuh"),
           os.path.join(HERE, "..", "include", "b200gsr.h"), os.path.join(HERE, "..", "include", "b200gsr_scene.h")]
NVCC_FLAGS = ["-gencode", "arch=compute_90a,code=sm_90a", "-O3", "-lineinfo", "-std=c++17",
              "-Xcompiler", "-fPIC", "--expt-relaxed-constexpr"]


def _nvcc() -> str:
    for cand in (os.environ.get("NVCC"), shutil.which("nvcc"), "/usr/local/cuda/bin/nvcc"):
        if cand and os.path.exists(cand):
            return cand
    raise RuntimeError("nvcc not found: cannot build libb200gsr.so")


# Build variants.  "default" is the product (libb200gsr.so).  "exact" (-DGSR_EXACT_EXP ->
# libb200gsr_exact.so) is the parity-diagnostic build: expf + IEEE division + the CPU checker's operation
# order in the blend exponent; selected with B200GSR_LIB=<path> by tools/parity_stats.py only.
VARIANTS = {"default": (LIB, []), "exact": (os.path.join(HERE, "libb200gsr_exact.so"), ["-DGSR_EXACT_EXP"])}


def needs_build(variant: str = "default") -> bool:
    lib = VARIANTS[variant][0]
    if not os.path.exists(lib):
        return True
    t = os.path.getmtime(lib)
    deps = [os.path.join(CSRC, s) for s in SOURCES] + HEADERS
    return any(os.path.getmtime(d) > t for d in deps)


def build(force: bool = False, verbose: bool = False, variant: str = "default", extra_flags=()) -> str:
    lib, defs = VARIANTS[variant]
    if not force and not extra_flags and not needs_build(variant):
        return lib
    nvcc = _nvcc()
    objdir = os.path.join(HERE, "build", variant)
    os.makedirs(objdir, exist_ok=True)
    objs = []
    procs = []
    for s in SOURCES:
        o = os.path.join(objdir, s.replace(".cu", ".o"))
        cmd = [nvcc, *NVCC_FLAGS, *defs, *extra_flags, "-c", os.path.join(CSRC, s), "-o", o]
        if verbose:
            cmd.insert(1, "-Xptxas=-v")
        procs.append((s, subprocess.Popen(cmd, stdout=subprocess.PIPE, stderr=subprocess.STDOUT, text=True)))
        objs.append(o)
    for s, p in procs:
        out, _ = p.communicate()
        if verbose and out:
            print(out, file=sys.stderr)
        if p.returncode != 0:
            raise RuntimeError(f"nvcc failed on {s}:\n{out}")
    link = [nvcc, "-shared", "-gencode", "arch=compute_90a,code=sm_90a", "-o", lib + ".tmp", *objs, "-ldl"]
    r = subprocess.run(link, stdout=subprocess.PIPE, stderr=subprocess.STDOUT, text=True)
    if r.returncode != 0:
        raise RuntimeError(f"link failed:\n{r.stdout}")
    os.replace(lib + ".tmp", lib)
    return lib


def build_all(force: bool = False, verbose: bool = False):
    return [build(force=force, verbose=verbose, variant=v) for v in VARIANTS]


if __name__ == "__main__":
    variants = [v for v in VARIANTS if f"--{v}" in sys.argv] or (list(VARIANTS) if "--all" in sys.argv else ["default"])
    for v in variants:
        print(build(force="--force" in sys.argv, verbose="-v" in sys.argv, variant=v))
