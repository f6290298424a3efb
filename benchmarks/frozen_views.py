#!/usr/bin/env python
"""Frozen groups on the two-step scene route: assemble_scene(frozen=) + rasterize_views(frozen_rows=) against the same
two ops without freezing, forward + backward of one training step's views.

Layout: harness/room.py::build_scene (env 2.0 M, floor 0.3 M, 4 objects of 0.08 M; M = 4, sh_degree 1),
4 views of 512 x 512 inside the room, SH and scale augmentation on in every view.  Configurations, after DreamScene's
scene stages (benchmarks/frozen_step.py):
  all   : every group trains; frozen = [False] * 6, which runs the plain kernels
  env   : stage 1, only env trains
  floor : stage 2, only floor trains
Noise modes: "fused" (in-kernel Philox, the two-op row of benchmarks/scene_render.py) and "torch" (torch.randn in the
reference's order, the reason to use this route).
Variants per (configuration, noise), alternating step by step:
  plain  : assemble_scene + rasterize_views, every group's gradient computed; the untrained ones are dropped
  frozen : the same with frozen= / frozen_rows=
Reported per variant: the median and p10 / p90 of the step time (CUDA events from the first op of the forward to the
end of the backward), peak allocated memory over a step above what was held before it, and the per-kernel device
time of one step (torch.profiler, a run of its own) for composite_bwd, project_bwd and assemble.  Prints one JSON line
per (configuration, noise) with the card's name, power limit and max SM clock read in the same run.

  python benchmarks/frozen_views.py [--steps 30] [--warmup 5] [--configs all,env,floor] [--noise fused,torch]
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
from dreamscene_b200.multiview import rasterize_views  # noqa: E402
from dreamscene_b200.scene import assemble_scene, frozen_rows  # noqa: E402
import scene_render  # noqa: E402

TRAINED = {"all": None, "env": 0, "floor": 1}     # group index trained by the stage (None: all of them)


def step(groups, S, target, seed, noise, frozen):
    B = len(S)
    gen = torch.Generator(device="cuda").manual_seed(seed) if noise == "torch" else None
    xyz, opac, scales_v, rots, shs_v = assemble_scene(groups, noise=noise, seed=seed, generator=gen, views=B,
                                                      frozen=frozen)
    outs = rasterize_views(S, xyz, opac, shs=list(shs_v.unbind(0)), scales=list(scales_v.unbind(0)), rotations=rots,
                           frozen_rows=None if frozen is None else frozen_rows(groups, frozen))
    images = torch.stack([o[0] for o in outs])
    depth = torch.stack([o[2][0] for o in outs])
    (((images - target) ** 2).mean() * 100 + depth.mean() * 0.1).backward()
    return images


def kernel_times(run):
    from torch.profiler import ProfilerActivity, profile
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        run()
        torch.cuda.synchronize()
    out = {}
    for e in prof.key_averages():
        if e.device_time_total > 0:
            name = e.key.replace("(anonymous namespace)::", "").replace("void ", "").split("<")[0].split("(")[0]
            out[name] = out.get(name, 0.0) + e.device_time_total / 1e3
    keep = ("composite_bwd", "project_bwd", "assemble")
    return {k: round(v, 4) for k, v in sorted(out.items()) if any(s in k for s in keep)}


def run_config(name, noise, groups, cams, deg, args, dev):
    trained = TRAINED[name]
    frozen = [trained is not None and i != trained for i in range(len(groups))]
    params = [t for g in groups for t in g.values()]
    bg = torch.ones(3, device=dev)
    target = torch.rand(4, 3, 512, 512, device=dev, generator=torch.Generator(device=dev).manual_seed(0))
    all_S = {it: scene_render.settings(cams(it), deg, bg) for it in range(args.warmup + args.steps)}
    variants = {"plain": None, "frozen": frozen}

    def clear():
        for p in params:
            p.grad = None

    # same images, and the trained groups' gradients within float atomics' rounding
    ref = {}
    for v, fz in variants.items():
        clear()
        img = step(groups, all_S[0], target, 3, noise, fz).detach()
        ref[v] = (img, [None if p.grad is None else p.grad.clone() for p in params])
    same_images = bool(torch.equal(ref["plain"][0], ref["frozen"][0]))
    rel = 0.0
    for a, b in zip(ref["plain"][1], ref["frozen"][1]):
        if b is not None and a.numel():
            rel = max(rel, float((a - b).double().norm() / a.double().norm().clamp_min(1e-30)))
    del ref
    times = {v: [] for v in variants}
    ev = [torch.cuda.Event(enable_timing=True) for _ in range(2)]
    order = list(variants)
    for it in range(args.warmup + args.steps):
        for v in (order if it % 2 == 0 else order[::-1]):
            clear()
            torch.cuda.synchronize()
            ev[0].record()
            step(groups, all_S[it], target, 100 + it, noise, variants[v])
            ev[1].record()
            torch.cuda.synchronize()
            if it >= args.warmup:
                times[v].append(ev[0].elapsed_time(ev[1]))
    peak, kern = {}, {}
    for v, fz in variants.items():
        clear()
        torch.cuda.synchronize()
        base = torch.cuda.memory_allocated()
        torch.cuda.reset_peak_memory_stats()
        step(groups, all_S[0], target, 5, noise, fz)
        torch.cuda.synchronize()
        peak[v] = round((torch.cuda.max_memory_allocated() - base) / 2 ** 20, 1)
        clear()
        kern[v] = kernel_times(lambda: step(groups, all_S[0], target, 7, noise, fz))
    clear()
    med = {v: float(np.median(times[v])) for v in variants}
    P = sum(int(g["_xyz"].shape[0]) for g in groups)
    nf = sum(int(g["_xyz"].shape[0]) for g, f in zip(groups, frozen) if f)
    return {"config": name, "noise": noise, "P": P, "frozen_rows": nf, "views": 4, "size": 512,
            "same_images": same_images, "trained_grad_max_rel": rel,
            "fwd_bwd_ms_median": {v: round(med[v], 4) for v in variants},
            "fwd_bwd_ms_p10_p90": {v: [round(float(np.percentile(times[v], q)), 4) for q in (10, 90)] for v in variants},
            "saving_ms": round(med["plain"] - med["frozen"], 4),
            "peak_allocated_MiB": peak, "kernel_ms": kern}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--steps", type=int, default=30)
    ap.add_argument("--warmup", type=int, default=5)
    ap.add_argument("--configs", default="all,env,floor")
    ap.add_argument("--noise", default="fused,torch")
    a = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("frozen_views.py measures on the GPU; no CUDA device found")
    dev = torch.device("cuda", 0)
    torch.manual_seed(0)
    info = scene_render.gpu_info()
    groups, cams, deg = scene_render.scene_layout(dev)
    groups = [{k: v.detach().requires_grad_(True) for k, v in g.items()} for g in groups]
    for noise in a.noise.split(","):
        for name in a.configs.split(","):
            res = run_config(name, noise, groups, cams, deg, a, dev)
            res["gpu"] = info
            print(json.dumps(res), flush=True)
            torch.cuda.empty_cache()


if __name__ == "__main__":
    main()
