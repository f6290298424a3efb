#!/usr/bin/env python
"""Densification statistics on the two-step scene route: rasterize_views(densify_stats=) against the eager statistics
after the backward, one training step's forward + backward + statistics.

Layouts (benchmarks/scene_render.py): object (1.2 M Gaussians, M = 16, sh_degree 3; its one group trains) and scene
(cfg5: env, floor and 4 objects, 2.63 M, M = 4, sh_degree 1), 4 views of 512 x 512, SH and scale augmentation on.
The scene layout runs DreamScene's scene stages: env (stage 1, only env trains), floor (stage 2) and both (stage 3);
the other groups are frozen (assemble_scene(frozen=) + rasterize_views(frozen_rows=)).  Noise modes "torch" (the
reference's torch.randn stream, the reason to use this route) and "fused".
Variants per (layout, stage, noise), alternating step by step:
  eager    : B means2D ports; after the backward one densify.add_densification_stats per trained group over its rows
             of view B-1's port gradient and radii (the reference's add_densification_stats_div slicing)
  backward : rasterize_views(densify_stats=stats_rows(...)), no ports: gathered inside the backward
Reported per variant: the median and p10 / p90 of the step time (CUDA events from the first op of the forward to the
end of the statistics), peak allocated memory over a step above what was held before it, and the device time of the
project_bwd_kernel launches of one step (torch.profiler, a run of its own).  Also whether the two variants' statistics
agree after one step from equal starting values (denom and max_radii2D exactly, accum within float atomics'
rounding).  Prints one JSON line per (layout, stage, noise) with the card's name, power limit and max SM clock read in
the same run.

  python benchmarks/views_stats_step.py [--steps 20] [--warmup 5] [--layouts object,scene] [--noise torch,fused]
"""
import argparse
import json
import os
import sys

import numpy as np
import torch

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, os.path.dirname(HERE))
sys.path.insert(0, HERE)
from dreamscene_b200 import densify  # noqa: E402
from dreamscene_b200.multiview import rasterize_views  # noqa: E402
from dreamscene_b200.scene import assemble_scene, frozen_rows, stats_rows  # noqa: E402
import scene_render  # noqa: E402

# stage -> trained group indices (scene layout: 0 = env, 1 = floor; object layout: its one group)
STAGES = {"scene": {"env": [0], "floor": [1], "both": [0, 1]}, "object": {"all": [0]}}


def step(groups, S, target, seed, noise, frozen, stats, backward):
    B = len(S)
    P = sum(int(g["_xyz"].shape[0]) for g in groups)
    gen = torch.Generator(device="cuda").manual_seed(seed) if noise == "torch" else None
    xyz, opac, scales_v, rots, shs_v = assemble_scene(groups, noise=noise, seed=seed, generator=gen, views=B,
                                                      frozen=frozen)
    m2d = None if backward else [torch.zeros(P, 3, device="cuda", requires_grad=True) for _ in range(B)]
    outs = rasterize_views(S, xyz, opac, shs=list(shs_v.unbind(0)), scales=list(scales_v.unbind(0)), rotations=rots,
                           means2D=m2d, frozen_rows=frozen_rows(groups, frozen),
                           densify_stats=stats_rows(groups, stats) if backward else None)
    images = torch.stack([o[0] for o in outs])
    depth = torch.stack([o[2][0] for o in outs])
    (((images - target) ** 2).mean() * 100 + depth.mean() * 0.1).backward()
    if not backward:
        lo = 0
        for g, st in zip(groups, stats):
            n = int(g["_xyz"].shape[0])
            if st is not None:
                densify.add_densification_stats(m2d[B - 1].grad[lo:lo + n], outs[B - 1][1][lo:lo + n], *st)
            lo += n


def project_bwd_ms(run):
    from torch.profiler import ProfilerActivity, profile
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        run()
        torch.cuda.synchronize()
    return round(sum(e.device_time_total for e in prof.key_averages()
                     if e.device_time_total > 0 and "project_bwd_kernel" in e.key) / 1e3, 4)


def new_stats(groups, trained, dev):
    return [(torch.zeros(int(g["_xyz"].shape[0]), 1, device=dev), torch.zeros(int(g["_xyz"].shape[0]), 1, device=dev),
             torch.zeros(int(g["_xyz"].shape[0]), device=dev)) if i in trained else None
            for i, g in enumerate(groups)]


def run_config(layout, stage, noise, groups, cams, deg, args, dev):
    trained = STAGES[layout][stage]
    frozen = [i not in trained for i in range(len(groups))]
    params = [t for g in groups for t in g.values()]
    bg = torch.ones(3, device=dev)
    target = torch.rand(4, 3, 512, 512, device=dev, generator=torch.Generator(device=dev).manual_seed(0))
    all_S = {it: scene_render.settings(cams(it), deg, bg) for it in range(args.warmup + args.steps)}
    variants = {"eager": False, "backward": True}
    stats = {v: new_stats(groups, trained, dev) for v in variants}

    def clear():
        for p in params:
            p.grad = None

    # one step from zero statistics: the two variants agree
    for v, bw in variants.items():
        clear()
        step(groups, all_S[0], target, 3, noise, frozen, stats[v], bw)
    acc_rel, exact = 0.0, True
    for a, b in zip(stats["eager"], stats["backward"]):
        if a is not None:
            acc_rel = max(acc_rel, float((a[0] - b[0]).double().norm() / a[0].double().norm().clamp_min(1e-30)))
            exact = exact and bool(torch.equal(a[1], b[1]) and torch.equal(a[2], b[2]))
    times = {v: [] for v in variants}
    ev = [torch.cuda.Event(enable_timing=True) for _ in range(2)]
    order = list(variants)
    for it in range(args.warmup + args.steps):
        for v in (order if it % 2 == 0 else order[::-1]):
            clear()
            torch.cuda.synchronize()
            ev[0].record()
            step(groups, all_S[it], target, 100 + it, noise, frozen, stats[v], variants[v])
            ev[1].record()
            torch.cuda.synchronize()
            if it >= args.warmup:
                times[v].append(ev[0].elapsed_time(ev[1]))
    peak, pbwd = {}, {}
    for v, bw in variants.items():
        clear()
        torch.cuda.synchronize()
        base = torch.cuda.memory_allocated()
        torch.cuda.reset_peak_memory_stats()
        step(groups, all_S[0], target, 5, noise, frozen, stats[v], bw)
        torch.cuda.synchronize()
        peak[v] = round((torch.cuda.max_memory_allocated() - base) / 2 ** 20, 1)
        clear()
        pbwd[v] = project_bwd_ms(lambda: step(groups, all_S[0], target, 7, noise, frozen, stats[v], bw))
    clear()
    med = {v: float(np.median(times[v])) for v in variants}
    P = sum(int(g["_xyz"].shape[0]) for g in groups)
    return {"layout": layout, "stage": stage, "noise": noise, "P": P, "views": 4, "size": 512,
            "stats_denom_max_radii_equal": exact, "stats_accum_max_rel": acc_rel,
            "step_ms_median": {v: round(med[v], 4) for v in variants},
            "step_ms_p10_p90": {v: [round(float(np.percentile(times[v], q)), 4) for q in (10, 90)] for v in variants},
            "saving_ms": round(med["eager"] - med["backward"], 4),
            "peak_allocated_MiB": peak, "project_bwd_ms": pbwd}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--steps", type=int, default=20)
    ap.add_argument("--warmup", type=int, default=5)
    ap.add_argument("--layouts", default="object,scene")
    ap.add_argument("--noise", default="torch,fused")
    a = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("views_stats_step.py measures on the GPU; no CUDA device found")
    dev = torch.device("cuda", 0)
    torch.manual_seed(0)
    info = scene_render.gpu_info()
    for layout in a.layouts.split(","):
        groups, cams, deg = (scene_render.scene_layout if layout == "scene" else scene_render.object_layout)(dev)
        groups = [{k: v.detach().requires_grad_(True) for k, v in g.items()} for g in groups]
        for noise in a.noise.split(","):
            for stage in STAGES[layout]:
                res = run_config(layout, stage, noise, groups, cams, deg, a, dev)
                res["gpu"] = info
                print(json.dumps(res), flush=True)
                torch.cuda.empty_cache()
        del groups
        torch.cuda.empty_cache()


if __name__ == "__main__":
    main()
