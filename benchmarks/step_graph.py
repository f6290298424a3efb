#!/usr/bin/env python
"""A whole training step, eager against StepGraph (two CUDA graphs with the loss eager between them).

  eager : render_scene(groups, S, return_scales=True) + disparity_from_depth_alpha + loss + backward
          + GaussianAdam.step() per group
  graph : sg.render(S) + the same loss + backward + sg.step()

The loss is an L2 against a fixed target, a total-variation term, a disparity term and the scale loss.  Both variants
change the cameras, flags, seed and the xyz lr every step, as a schedule does.  Layouts (benchmarks/scene_render.py):
  object : 1.2 M Gaussians in one group, M = 16, 4 views of 512 x 512
  scene  : harness/room.py::build_scene (cfg5: 2.63 M Gaussians in 6 groups, M = 4), 4 views of 512 x 512

Per variant, alternating the variants in rounds:
  sync_ms    : median wall time of one step followed by torch.cuda.synchronize()
  b2b_ms     : wall time per step of `steps` back-to-back steps with one synchronize at the end
  host_us    : host time per step in the back-to-back run (until the last call returns, before the synchronize)
  device_ms  : summed CUDA kernel and copy time per step from torch.profiler, and within it the project_sh and
               project_bwd kernels (graph: the DYN instantiations, eager: the by-value RAW ones)
  capture_ms : the graph's first step (eager measurement + capture + the first replay), timed after one eager step
               has initialised the library and the allocator
Prints one JSON line per layout.

  python benchmarks/step_graph.py [--steps 20] [--rounds 5] [--layouts object,scene]
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


def clone(groups):
    return [{k: v.detach().clone().requires_grad_(True) for k, v in g.items()} for g in groups]


def optimizers(groups):
    return [GaussianAdam([{"params": [g[k]], "lr": LRS[k]} for k in NAMES], lr=0.0, eps=1e-15) for g in groups]


def loss_fn(image, disp, scales, target):
    tv = (image[..., 1:, :] - image[..., :-1, :]).abs().mean() + (image[..., :, 1:] - image[..., :, :-1]).abs().mean()
    return ((image - target) ** 2).mean() + 0.1 * tv + 0.01 * disp.mean() + scales.mean()


class Eager:
    def __init__(self, groups):
        self.groups, self.opts = groups, optimizers(groups)

    def step(self, S, it, target):
        for o in self.opts:
            o.param_groups[0]["lr"] = LRS["_xyz"] * 0.99 ** it
        flags = [(v + it) % 2 == 0 for v in range(len(S))]
        outs, scales = render_scene(self.groups, S, shs_aug=flags, scale_aug=flags, seed=it, return_scales=True)
        image = torch.stack([o[0] for o in outs])
        disp, _ = disparity_from_depth_alpha(torch.stack([o[2] for o in outs]),
                                             [1.0 / (2.0 * float(s.tanfovx)) for s in S])
        loss_fn(image, disp, scales, target).backward()
        for o in self.opts:
            o.step()
            o.zero_grad()


class Graph:
    def __init__(self, groups, B):
        self.groups, self.opts = groups, optimizers(groups)
        self.sg = StepGraph(groups, self.opts, views=B, height=512, width=512)

    def step(self, S, it, target):
        for o in self.opts:
            o.param_groups[0]["lr"] = LRS["_xyz"] * 0.99 ** it
        flags = [(v + it) % 2 == 0 for v in range(len(S))]
        out = self.sg.render(S, shs_aug=flags, scale_aug=flags, seed=it)
        loss_fn(out.image, out.disp, out.scales, target).backward()
        self.sg.step()


def device_ms(run, steps):
    """-> (all kernels and copies, project_sh kernels, project_bwd kernels) in ms per step."""
    from torch.autograd import DeviceType
    with torch.profiler.profile(activities=[torch.profiler.ProfilerActivity.CUDA]) as prof:
        for _ in range(steps):
            run()
        torch.cuda.synchronize()
    ev = [e for e in prof.events() if e.device_type == DeviceType.CUDA]
    tot = lambda pred: round(sum(e.self_device_time_total for e in ev if pred(e.name)) / 1e3 / steps, 4)
    return tot(lambda n: True), tot(lambda n: "project_sh_kernel" in n), tot(lambda n: "project_bwd_kernel" in n)


def run_layout(name, args, dev):
    groups, cams, deg = scene_render.object_layout(dev) if name == "object" else scene_render.scene_layout(dev)
    bg = torch.zeros(3, device=dev)
    S_of = lambda it: scene_render.settings(cams(it), deg, bg)
    target = torch.rand(4, 3, 512, 512, device=dev, generator=torch.Generator(device=dev).manual_seed(0))
    variants = {"eager": Eager(clone(groups)), "graph": Graph(clone(groups), 4)}
    del groups
    res = {k: {"sync_ms": [], "b2b_ms": [], "host_us": []} for k in variants}
    variants["eager"].step(S_of(0), 0, target)  # one-time library / allocator initialisation, untimed
    torch.cuda.synchronize()
    t0 = time.perf_counter()
    variants["graph"].step(S_of(1), 1, target)  # measurement + capture + first replay
    torch.cuda.synchronize()
    capture_ms = round((time.perf_counter() - t0) * 1e3, 2)
    it = 2
    for _ in range(args.warmup):
        for v in variants.values():
            v.step(S_of(it), it, target)
            it += 1
    variants["graph"].sg.check()
    settings = [S_of(j) for j in range(args.steps)]
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
            t1 = time.perf_counter()
            torch.cuda.synchronize()
            t2 = time.perf_counter()
            res[k]["b2b_ms"].append((t2 - t0) * 1e3 / args.steps)
            res[k]["host_us"].append((t1 - t0) * 1e6 / args.steps)
            it += args.steps
    variants["graph"].sg.check()
    out = {"layout": name, "views": 4, "size": 512,
           "P": sum(int(g["_xyz"].shape[0]) for g in variants["eager"].groups)}
    for k, v in variants.items():
        r = res[k]
        med = lambda xs: round(sorted(xs)[len(xs) // 2], 4)
        dev_ms, sh_ms, bwd_ms = device_ms(lambda: v.step(settings[0], it, target), 5)
        out[k] = {"sync_ms": med(r["sync_ms"]), "b2b_ms": med(r["b2b_ms"]), "b2b_ms_range": [round(min(r["b2b_ms"]), 4),
                  round(max(r["b2b_ms"]), 4)], "host_us": round(sorted(r["host_us"])[len(r["host_us"]) // 2], 1),
                  "device_ms": dev_ms, "project_sh_ms": sh_ms, "project_bwd_ms": bwd_ms}
    out["graph"]["capture_ms"] = capture_ms
    return out


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--steps", type=int, default=20)
    ap.add_argument("--warmup", type=int, default=3)
    ap.add_argument("--rounds", type=int, default=5)
    ap.add_argument("--layouts", default="object,scene")
    a = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("step_graph.py measures on the GPU; no CUDA device found")
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
