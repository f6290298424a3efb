#!/usr/bin/env python
"""Frozen parameter groups (DESIGN.md f11) on the scene layout: a training step that trains some groups and renders
all of them, with the frozen groups' backward skipped (frozen=) against the plain backward that computes every
group's gradients and steps only the trained groups' optimizers.

Layout: harness/room.py::build_scene (env 2.0 M, floor 0.3 M, 4 objects of 0.08 M; M = 4, sh_degree 1),
4 views of 512 x 512.  Configurations, after DreamScene's scene stages:
  all   : every group trains (scene_optim); frozen=[False] * 6 is the plain backward
  env   : stage 1, only env trains
  floor : stage 2, only floor trains
Variants per configuration, alternating in rounds:
  eager_plain / eager_frozen : render_scene(return_scales=True) + disparity + loss + backward + the trained groups'
                               GaussianAdam.step(); the loss is an L2 against a fixed target plus the regularisers
                               tv(image) * 1 and mean(mean(scales, -1)) * 0.5, as torch expressions
  graph_plain / graph_frozen : StepGraph(tv_weight=1, tv_depth_weight=0, scale_weight=0.5) with the L2 eager
Reported per variant:
  sync_ms   : median wall time of one step followed by torch.cuda.synchronize()
  b2b_ms    : wall time per step of `steps` back-to-back steps with one synchronize at the end (median over rounds)
  device_ms : summed CUDA kernel and copy time per step (torch.profiler, a run of its own), and within it the
              project_bwd and composite_bwd kernels
  peak_mb   : peak allocated memory of building the variant and running its first two steps, above what was
              allocated before (the graph's static buffers and the optimizer state included)
Prints one JSON line per configuration with the card's name, power limit and max SM clock read in the same run.

  python benchmarks/frozen_step.py [--steps 20] [--warmup 3] [--rounds 5] [--configs all,env,floor]
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
from dreamscene_b200.postprocess import disparity_from_depth_alpha  # noqa: E402
from dreamscene_b200.scene import render_scene  # noqa: E402
import scene_render  # noqa: E402

NAMES = scene_render.NAMES
LRS = {"_xyz": 1.6e-4, "_opacity": 0.05, "_scaling": 0.005, "_rotation": 0.001, "_features_dc": 0.0025,
       "_features_rest": 0.000125}
TRAINED = {"all": None, "env": 0, "floor": 1}     # group index trained by the stage (None: all of them)
TV_W, SCALE_W = 1.0, 0.5


def clone(groups):
    return [{k: v.detach().clone().requires_grad_(True) for k, v in g.items()} for g in groups]


def optimizers(groups, trained):
    return [GaussianAdam([{"params": [g[k]], "lr": LRS[k]} for k in NAMES], lr=0.0, eps=1e-15)
            for i, g in enumerate(groups) if trained is None or i == trained]


def tv(x):
    return (x[..., 1:, :] - x[..., :-1, :]).abs().mean() + (x[..., :, 1:] - x[..., :, :-1]).abs().mean()


class Eager:
    def __init__(self, groups, trained, frozen):
        self.groups, self.opts, self.frozen = groups, optimizers(groups, trained), frozen

    def step(self, S, it, target):
        flags = [(v + it) % 2 == 0 for v in range(len(S))]
        outs, scales = render_scene(self.groups, S, shs_aug=flags, scale_aug=flags, seed=it, return_scales=True,
                                    frozen=self.frozen)
        image = torch.stack([o[0] for o in outs])
        disp, _ = disparity_from_depth_alpha(torch.stack([o[2] for o in outs]),
                                             [1.0 / (2.0 * float(s.tanfovx)) for s in S])
        loss = ((image - target) ** 2).mean() + 0.01 * disp.mean()
        (loss + TV_W * tv(image) + SCALE_W * scales.mean(-1).mean()).backward()
        for o in self.opts:
            o.step()
            o.zero_grad()
        for g in self.groups:                 # the untrained groups' gradients (plain backward) are dropped
            for t in g.values():
                t.grad = None


class Graph:
    def __init__(self, groups, trained, frozen, B):
        self.groups, self.opts = groups, optimizers(groups, trained)
        self.sg = StepGraph(groups, self.opts, views=B, height=512, width=512, tv_weight=TV_W, tv_depth_weight=0.0,
                            scale_weight=SCALE_W, frozen=frozen)

    def step(self, S, it, target):
        flags = [(v + it) % 2 == 0 for v in range(len(S))]
        out = self.sg.render(S, shs_aug=flags, scale_aug=flags, seed=it)
        (((out.image - target) ** 2).mean() + 0.01 * out.disp.mean()).backward()
        self.sg.step()


def device_ms(run, steps):
    """-> (all kernels and copies, project_bwd kernels, composite_bwd kernels) in ms per step."""
    from torch.autograd import DeviceType
    with torch.profiler.profile(activities=[torch.profiler.ProfilerActivity.CUDA]) as prof:
        for _ in range(steps):
            run()
        torch.cuda.synchronize()
    ev = [e for e in prof.events() if e.device_type == DeviceType.CUDA]
    tot = lambda pred: round(sum(e.self_device_time_total for e in ev if pred(e.name)) / 1e3 / steps, 4)
    return (tot(lambda n: True), tot(lambda n: "project_bwd_kernel" in n), tot(lambda n: "composite_bwd_kernel" in n))


def run_config(name, args, dev, base_groups, cams, deg):
    trained = TRAINED[name]
    ng = len(base_groups)
    frozen = [trained is not None and i != trained for i in range(ng)]
    bg = torch.zeros(3, device=dev)
    S_of = lambda it: scene_render.settings(cams(it), deg, bg)
    target = torch.rand(4, 3, 512, 512, device=dev, generator=torch.Generator(device=dev).manual_seed(0))
    makers = {"eager_plain": lambda g: Eager(g, trained, None), "eager_frozen": lambda g: Eager(g, trained, frozen),
              "graph_plain": lambda g: Graph(g, trained, None, 4), "graph_frozen": lambda g: Graph(g, trained, frozen, 4)}
    variants, peak = {}, {}
    it = 0
    for k, make in makers.items():
        torch.cuda.synchronize()
        torch.cuda.reset_peak_memory_stats(dev)
        before = torch.cuda.memory_allocated(dev)
        v = variants[k] = make(clone(base_groups))
        for _ in range(2):                  # library / allocator set-up and, for the graphs, the capture
            v.step(S_of(it), it, target)
            it += 1
        torch.cuda.synchronize()
        peak[k] = round((torch.cuda.max_memory_allocated(dev) - before) / 2 ** 20, 1)
    for _ in range(args.warmup):
        for v in variants.values():
            v.step(S_of(it), it, target)
            it += 1
    settings = [S_of(j) for j in range(args.steps)]
    res = {k: {"sync_ms": [], "b2b_ms": []} for k in variants}
    for _ in range(args.rounds):
        for k, v in variants.items():            # alternate the variants
            for j in range(args.steps):
                torch.cuda.synchronize()
                t0 = time.perf_counter()
                v.step(settings[j], it + j, target)
                torch.cuda.synchronize()
                res[k]["sync_ms"].append((time.perf_counter() - t0) * 1e3)
            torch.cuda.synchronize()
            t0 = time.perf_counter()
            for j in range(args.steps):
                v.step(settings[j], it + j, target)
            torch.cuda.synchronize()
            res[k]["b2b_ms"].append((time.perf_counter() - t0) * 1e3 / args.steps)
            it += args.steps
    for k in ("graph_plain", "graph_frozen"):
        variants[k].sg.check()
    med = lambda xs: round(sorted(xs)[len(xs) // 2], 4)
    rows = sum(int(g["_xyz"].shape[0]) for g in base_groups)
    frozen_rows = sum(int(g["_xyz"].shape[0]) for g, f in zip(base_groups, frozen) if f)
    out = {"config": name, "views": 4, "size": 512, "P": rows, "frozen_rows": frozen_rows, "frozen": frozen}
    for k, v in variants.items():
        dev_ms, pbwd, cbwd = device_ms(lambda: v.step(settings[0], it, target), 5)
        out[k] = {"sync_ms": med(res[k]["sync_ms"]), "b2b_ms": med(res[k]["b2b_ms"]),
                  "b2b_ms_range": [round(min(res[k]["b2b_ms"]), 4), round(max(res[k]["b2b_ms"]), 4)],
                  "device_ms": dev_ms, "project_bwd_ms": pbwd, "composite_bwd_ms": cbwd, "peak_mb": peak[k]}
    return out


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--steps", type=int, default=20)
    ap.add_argument("--warmup", type=int, default=3)
    ap.add_argument("--rounds", type=int, default=5)
    ap.add_argument("--configs", default="all,env,floor")
    a = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("frozen_step.py measures on the GPU; no CUDA device found")
    dev = torch.device("cuda", 0)
    torch.manual_seed(0)
    info = scene_render.gpu_info()
    groups, cams, deg = scene_render.scene_layout(dev)
    groups = [{k: v.detach() for k, v in g.items()} for g in groups]
    for name in a.configs.split(","):
        res = run_config(name, a, dev, groups, cams, deg)
        res["gpu"] = info
        print(json.dumps(res), flush=True)
        torch.cuda.empty_cache()


if __name__ == "__main__":
    main()
