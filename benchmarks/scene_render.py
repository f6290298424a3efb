#!/usr/bin/env python
"""render_scene against the two-op path it replaces, forward + backward of one training step's views.

  two_op : xyz, opac, scales_v, rots, shs_v = assemble_scene(groups, noise="fused", views=B)
           rasterize_views(S, xyz, opac, shs=list(shs_v), scales=list(scales_v), rotations=rots)
  scene  : render_scene(groups, S)                  (activations + augmentation inside project_sh / project_bwd)

Both with SH and scale augmentation on in every view and the same seed, so both render the same images.  Layouts:
  object : 1.2 M Gaussians in one group, M = 16 (sh_degree 3), 4 views of 512 x 512 (object_render)
  scene  : benchmarks/scene_step.py::build_scene (2.63 M Gaussians in 6 groups, M = 4, sh_degree 1), 4 views of
           512 x 512 inside the room (scene_render)

Per layout the variants alternate step by step; a step is timed with CUDA events from the first op of the forward
to the end of the backward, and the median is reported.  Each variant's peak allocated memory over a step
(torch.cuda.max_memory_allocated above the memory held before it) is measured in a step of its own, and its kernel
times come from a torch.profiler run of one step, summed per kernel.  render_scene's calls are also recorded by the
library's stage timers (b200gsr_profile_*).  Prints one JSON line per layout.

  python benchmarks/scene_render.py [--steps 30] [--warmup 5] [--layouts object,scene]
"""
import argparse
import json
import math
import os
import subprocess
import sys

import numpy as np
import torch

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, os.path.dirname(HERE))
sys.path.insert(0, HERE)
from dreamscene_b200 import GaussianRasterizationSettings, _lib  # noqa: E402
from dreamscene_b200.multiview import rasterize_views  # noqa: E402
from dreamscene_b200.scene import assemble_scene, render_scene  # noqa: E402
from harness import cameras  # noqa: E402
import scene_step  # noqa: E402

NAMES = ("_xyz", "_opacity", "_scaling", "_rotation", "_features_dc", "_features_rest")


def object_layout(dev, P=1_200_000, M=16, seed=0):
    rng = np.random.RandomState(seed)
    d = rng.normal(size=(P, 3)); d /= np.linalg.norm(d, axis=1, keepdims=True)
    xyz = 0.5 * np.cbrt(rng.random_sample((P, 1))) * d
    g = scene_step.make_group(xyz, rng, M, dev, scale=0.004)
    group = {"_xyz": g["xyz"], "_opacity": g["opacity"], "_scaling": g["scaling"], "_rotation": g["rotation"],
             "_features_dc": g["f_dc"], "_features_rest": g["f_rest"]}
    cams = lambda it: [cameras.orbit_camera(radius=2.5, theta_deg=60.0 + 10 * math.sin(it + k), phi_deg=90.0 * k + 13 * it,
                                            fovx=0.8, height=512, width=512, device=dev) for k in range(4)]
    return [group], cams, 3


def scene_layout(dev):
    groups = [{"_xyz": g["xyz"], "_opacity": g["opacity"], "_scaling": g["scaling"], "_rotation": g["rotation"],
               "_features_dc": g["f_dc"], "_features_rest": g["f_rest"]} for g in scene_step.build_scene(dev)]
    cams = lambda it: [scene_step.scene_camera(it * 4 + k, 512, dev) for k in range(4)]
    return groups, cams, 1


def settings(cams, deg, bg):
    return [GaussianRasterizationSettings(
        image_height=c.image_height, image_width=c.image_width, tanfovx=c.tanfovx, tanfovy=c.tanfovy, bg=bg,
        scale_modifier=1.0, viewmatrix=c.world_view_transform, projmatrix=c.full_proj_transform, sh_degree=deg,
        campos=c.camera_center, prefiltered=False, score_flag=False) for c in cams]


def step(variant, groups, S, target, seed):
    B = len(S)
    if variant == "two_op":
        xyz, opac, scales_v, rots, shs_v = assemble_scene(groups, noise="fused", seed=seed, views=B)
        outs = rasterize_views(S, xyz, opac, shs=list(shs_v.unbind(0)), scales=list(scales_v.unbind(0)), rotations=rots)
    else:
        outs = render_scene(groups, S, seed=seed)
    images = torch.stack([o[0] for o in outs])
    depth = torch.stack([o[2][0] for o in outs])
    (((images - target) ** 2).mean() * 100 + depth.mean() * 0.1).backward()
    return images


def kernel_times(variant, groups, S, target):
    from torch.profiler import ProfilerActivity, profile
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        step(variant, groups, S, target, 7)
        torch.cuda.synchronize()
    out = {}
    for e in prof.key_averages():
        if e.device_time_total > 0:
            name = e.key.replace("(anonymous namespace)::", "").replace("void ", "").split("<")[0].split("(")[0]
            out[name] = out.get(name, 0.0) + e.device_time_total / 1e3
    return {k: round(v, 4) for k, v in sorted(out.items(), key=lambda kv: -kv[1]) if v >= 0.005}


def run_layout(name, groups, cams, deg, args, dev):
    params = [t for g in groups for t in g.values()]
    P = sum(int(g["_xyz"].shape[0]) for g in groups)
    M = 1 + int(groups[0]["_features_rest"].shape[1])
    bg = torch.ones(3, device=dev)
    target = torch.rand(4, 3, 512, 512, device=dev)
    all_S = {it: settings(cams(it), deg, bg) for it in range(args.warmup + args.steps)}
    variants = ("two_op", "scene")

    def clear():
        for p in params:
            p.grad = None

    # same images from the same seed: the two paths render the same thing
    clear()
    img = {v: step(v, groups, all_S[0], target, 3).detach() for v in variants}
    same_images = bool(torch.equal(img["two_op"], img["scene"]))
    clear()
    times = {v: [] for v in variants}
    ev = [torch.cuda.Event(enable_timing=True) for _ in range(2)]
    for it in range(args.warmup + args.steps):
        for v in (variants if it % 2 == 0 else variants[::-1]):
            clear()
            torch.cuda.synchronize()
            ev[0].record()
            step(v, groups, all_S[it], target, 100 + it)
            ev[1].record()
            torch.cuda.synchronize()
            if it >= args.warmup:
                times[v].append(ev[0].elapsed_time(ev[1]))
    peak = {}
    for v in variants:
        clear()
        torch.cuda.synchronize()
        base = torch.cuda.memory_allocated()
        torch.cuda.reset_peak_memory_stats()
        step(v, groups, all_S[0], target, 5)
        torch.cuda.synchronize()
        peak[v] = round((torch.cuda.max_memory_allocated() - base) / 2 ** 20, 1)
    kern = {}
    for v in variants:
        clear()
        kern[v] = kernel_times(v, groups, all_S[0], target)
    clear()
    _lib.profile_enable(4)
    step("scene", groups, all_S[0], target, 5)
    torch.cuda.synchronize()
    stages = {k: round(float(np.mean(x)), 4) for k, x in _lib.profile_collect().items() if x}
    _lib.profile_enable(0)
    med = {v: float(np.median(times[v])) for v in variants}
    B = 4
    return {"layout": name, "P": P, "M": M, "sh_degree": deg, "views": B, "size": 512,
            "same_images": same_images,
            "fwd_bwd_ms_median": {v: round(med[v], 4) for v in variants},
            "fwd_bwd_ms_p10_p90": {v: [round(float(np.percentile(times[v], q)), 4) for q in (10, 90)] for v in variants},
            "saving_ms": round(med["two_op"] - med["scene"], 4),
            "handoff_bytes_model_GB": round(4 * B * P * (3 * M + 3) * 4 / 1e9, 3),
            "peak_allocated_MiB": peak, "kernel_ms": kern, "render_scene_stage_ms": stages}


def gpu_info():
    try:
        out = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                             capture_output=True, text=True, timeout=30).stdout.strip().splitlines()
        return out[0] if out else None
    except Exception:      # noqa: BLE001 - informational only
        return None


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--steps", type=int, default=30)
    ap.add_argument("--warmup", type=int, default=5)
    ap.add_argument("--layouts", default="object,scene")
    a = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("scene_render.py measures on the GPU; no CUDA device found")
    dev = torch.device("cuda", 0)
    torch.manual_seed(0)
    info = gpu_info()
    for name in a.layouts.split(","):
        groups, cams, deg = object_layout(dev) if name == "object" else scene_layout(dev)
        res = run_layout(name, groups, cams, deg, a, dev)
        res["gpu"] = info
        print(json.dumps(res), flush=True)
        del groups
        torch.cuda.empty_cache()


if __name__ == "__main__":
    main()
