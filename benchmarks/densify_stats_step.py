#!/usr/bin/env python
"""Densification statistics inside the replayed step (DESIGN.md f12) against the eager statistics after it.

Layouts (benchmarks/scene_render.py): object (1.2 M Gaussians, M = 16, sh_degree 3) and scene (cfg5: env, floor and
4 objects, 2.63 M, M = 4, sh_degree 1), 4 views of 512 x 512.  Every group trains and gathers statistics.
Variants, alternating in rounds:
  eager : StepGraph(keep_means2D=True); after each step one densify.add_densification_stats per group on view B-1 of
          sg.d_means2D and out.radii (the reference's add_densification_stats)
  graph : StepGraph(densify_stats=..., keep_means2D=False); step(stats_view=-1) gathers them inside the backward graph,
          and no [B,P,3] d_means2D is written
The eager loss is an L2 against a fixed target plus 0.01 * mean(disp).
Reported per variant:
  b2b_ms         : wall time per step of `steps` back-to-back steps with one synchronize at the end (median over rounds)
  device_ms      : summed CUDA kernel and copy time per step (torch.profiler, a run of its own)
  project_bwd_ms : within it, the project_bwd_kernel launches (plain and STATS instantiations)
  peak_mb        : peak allocated memory of building the variant and running its first two steps, above what was
                   allocated before (the graph's static buffers, statistics and optimizer state included)
Prints one JSON line per layout with the card's name, power limit and max SM clock read in the same run.

  python benchmarks/densify_stats_step.py [--steps 20] [--warmup 3] [--rounds 5] [--layouts object,scene]
"""
import argparse
import json
import os
import sys
import time

import torch

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, os.path.dirname(HERE))
sys.path.insert(0, HERE)
from dreamscene_b200 import GaussianAdam, StepGraph  # noqa: E402
from dreamscene_b200 import densify  # noqa: E402
import scene_render  # noqa: E402

NAMES = scene_render.NAMES
LRS = {"_xyz": 1.6e-4, "_opacity": 0.05, "_scaling": 0.005, "_rotation": 0.001, "_features_dc": 0.0025,
       "_features_rest": 0.000125}


def clone(groups):
    return [{k: v.detach().clone().requires_grad_(True) for k, v in g.items()} for g in groups]


def optimizers(groups):
    return [GaussianAdam([{"params": [g[k]], "lr": LRS[k]} for k in NAMES], lr=0.0, eps=1e-15) for g in groups]


def new_stats(groups, dev):
    return [(torch.zeros(int(g["_xyz"].shape[0]), 1, device=dev), torch.zeros(int(g["_xyz"].shape[0]), 1, device=dev),
             torch.zeros(int(g["_xyz"].shape[0]), device=dev)) for g in groups]


class Variant:
    def __init__(self, groups, in_graph, dev):
        self.groups, self.opts, self.in_graph = groups, optimizers(groups), in_graph
        self.stats = new_stats(groups, dev)
        self.rows = []
        o = 0
        for g in groups:
            n = int(g["_xyz"].shape[0])
            self.rows.append((o, o + n))
            o += n
        self.sg = StepGraph(groups, self.opts, views=4, height=512, width=512,
                            densify_stats=self.stats if in_graph else None, keep_means2D=not in_graph)

    def step(self, S, it, target):
        flags = [(v + it) % 2 == 0 for v in range(len(S))]
        out = self.sg.render(S, shs_aug=flags, scale_aug=flags, seed=it)
        (((out.image - target) ** 2).mean() + 0.01 * out.disp.mean()).backward()
        self.sg.step(stats_view=-1)
        if not self.in_graph:
            v = len(S) - 1
            for (a, b), st in zip(self.rows, self.stats):
                densify.add_densification_stats(self.sg.d_means2D[v, a:b], out.radii[v, a:b], *st)


def device_ms(run, steps):
    """-> (all kernels and copies, project_bwd kernels) in ms per step."""
    from torch.autograd import DeviceType
    with torch.profiler.profile(activities=[torch.profiler.ProfilerActivity.CUDA]) as prof:
        for _ in range(steps):
            run()
        torch.cuda.synchronize()
    ev = [e for e in prof.events() if e.device_type == DeviceType.CUDA]
    tot = lambda pred: round(sum(e.self_device_time_total for e in ev if pred(e.name)) / 1e3 / steps, 4)
    return tot(lambda n: True), tot(lambda n: "project_bwd" in n)


def run_layout(name, args, dev):
    groups, cams, deg = scene_render.object_layout(dev) if name == "object" else scene_render.scene_layout(dev)
    groups = [{k: v.detach() for k, v in g.items()} for g in groups]
    bg = torch.zeros(3, device=dev)
    S_of = lambda it: scene_render.settings(cams(it), deg, bg)
    target = torch.rand(4, 3, 512, 512, device=dev, generator=torch.Generator(device=dev).manual_seed(0))
    P = sum(int(g["_xyz"].shape[0]) for g in groups)
    variants, peak = {}, {}
    it = 0
    for k in ("eager", "graph"):
        torch.cuda.synchronize()
        torch.cuda.reset_peak_memory_stats(dev)
        before = torch.cuda.memory_allocated(dev)
        v = variants[k] = Variant(clone(groups), k == "graph", dev)
        for _ in range(2):                  # library / allocator set-up and the capture
            v.step(S_of(it), it, target)
            it += 1
        torch.cuda.synchronize()
        peak[k] = round((torch.cuda.max_memory_allocated(dev) - before) / 2 ** 20, 1)
    del groups
    for _ in range(args.warmup):
        for v in variants.values():
            v.step(S_of(it), it, target)
            it += 1
    settings = [S_of(j) for j in range(args.steps)]
    res = {k: [] for k in variants}
    for _ in range(args.rounds):
        for k, v in variants.items():            # alternate the variants
            torch.cuda.synchronize()
            t0 = time.perf_counter()
            for j in range(args.steps):
                v.step(settings[j], it + j, target)
            torch.cuda.synchronize()
            res[k].append((time.perf_counter() - t0) * 1e3 / args.steps)
            it += args.steps
    for v in variants.values():
        v.sg.check()
    med = lambda xs: round(sorted(xs)[len(xs) // 2], 4)
    out = {"layout": name, "views": 4, "size": 512, "P": P}
    for k, v in variants.items():
        dev_ms, pbwd = device_ms(lambda: v.step(settings[0], it, target), 5)
        out[k] = {"b2b_ms": med(res[k]), "b2b_ms_range": [round(min(res[k]), 4), round(max(res[k]), 4)],
                  "device_ms": dev_ms, "project_bwd_ms": pbwd, "peak_mb": peak[k]}
    return out


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--steps", type=int, default=20)
    ap.add_argument("--warmup", type=int, default=3)
    ap.add_argument("--rounds", type=int, default=5)
    ap.add_argument("--layouts", default="object,scene")
    a = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("densify_stats_step.py measures on the GPU; no CUDA device found")
    dev = torch.device("cuda", 0)
    torch.manual_seed(0)
    info = scene_render.gpu_info()
    for name in a.layouts.split(","):
        res = run_layout(name, a, dev)
        res["gpu"] = info
        print(json.dumps(res), flush=True)
        torch.cuda.empty_cache()


if __name__ == "__main__":
    main()
