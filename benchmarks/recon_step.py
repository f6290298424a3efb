#!/usr/bin/env python
"""The refine stages' reconstruction step, one view per step: eager, StepGraph with the loss eager between the graphs,
and StepGraph in target mode (the loss inside the render graph).

  eager  : render_scene(groups, [view], no augmentation) + disparity_from_depth_alpha
           + l2_loss(image.half(), gt[i]) * 100 + backward + GaussianAdam.step() per group
  graph  : sg.render([view]) + the same torch loss on out.image + backward + sg.step()
  target : StepGraph(..., target=gt): sg.render([view], target_index=[i]) + sg.step()

The pseudo ground truth is G = 18 float16 images of 512 x 512 (the object stage's 18 views).  Every step changes the
camera, the target index and the xyz lr, as the refine loop does.  Layouts (benchmarks/scene_render.py):
  object : 1.2 M Gaussians in one group, M = 16
  scene  : harness/room.py::build_scene (cfg5: 2.63 M Gaussians in 6 groups, M = 4)

Per variant, alternating the variants in rounds:
  sync_ms    : median wall time of one step followed by torch.cuda.synchronize()
  b2b_ms     : wall time per step of `steps` back-to-back steps with one synchronize at the end
  host_us    : host time per step in the back-to-back run (until the last call returns, before the synchronize)
  device_ms  : summed CUDA kernel and copy time per step from torch.profiler, after the timed rounds and apart from
               them; for target also the recon_l2 kernels' share (recon_l2_ms)
  capture_ms : the graph's first step (eager measurement + capture + the first replay), timed after one eager step
               has initialised the library and the allocator
Prints one JSON line per layout.

  python benchmarks/recon_step.py [--steps 20] [--rounds 3] [--layouts object,scene]
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
G = 18


def clone(groups):
    return [{k: v.detach().clone().requires_grad_(True) for k, v in g.items()} for g in groups]


def optimizers(groups):
    return [GaussianAdam([{"params": [g[k]], "lr": LRS[k]} for k in NAMES], lr=0.0, eps=1e-15) for g in groups]


def l2_loss(image, gt):
    return ((image.to(torch.float16) - gt) ** 2).mean() * 100


class Eager:
    def __init__(self, groups, gt):
        self.groups, self.opts, self.gt = groups, optimizers(groups), gt

    def step(self, S, it):
        for o in self.opts:
            o.param_groups[0]["lr"] = LRS["_xyz"] * 0.99 ** it
        outs = render_scene(self.groups, S, shs_aug=False, scale_aug=False, seed=it)
        disparity_from_depth_alpha(outs[0][2], 1.0 / (2.0 * float(S[0].tanfovx)))
        l2_loss(outs[0][0], self.gt[it % G]).backward()
        for o in self.opts:
            o.step()
            o.zero_grad()


class Graph:
    def __init__(self, groups, gt, target_mode):
        self.groups, self.opts, self.gt, self.target_mode = groups, optimizers(groups), gt, target_mode
        kw = dict(target=gt, target_weight=100.0) if target_mode else {}
        self.sg = StepGraph(groups, self.opts, views=1, height=512, width=512, **kw)

    def step(self, S, it):
        for o in self.opts:
            o.param_groups[0]["lr"] = LRS["_xyz"] * 0.99 ** it
        if self.target_mode:
            self.sg.render(S, shs_aug=False, scale_aug=False, seed=it, target_index=[it % G])
        else:
            out = self.sg.render(S, shs_aug=False, scale_aug=False, seed=it)
            l2_loss(out.image[0], self.gt[it % G]).backward()
        self.sg.step()


def device_ms(run, steps):
    """-> (all kernels and copies, the recon_l2 kernels) in ms per step."""
    from torch.autograd import DeviceType
    with torch.profiler.profile(activities=[torch.profiler.ProfilerActivity.CUDA]) as prof:
        for _ in range(steps):
            run()
        torch.cuda.synchronize()
    ev = [e for e in prof.events() if e.device_type == DeviceType.CUDA]
    tot = lambda pred: round(sum(e.self_device_time_total for e in ev if pred(e.name)) / 1e3 / steps, 4)
    return tot(lambda n: True), tot(lambda n: "recon_l2" in n)


def run_layout(name, args, dev):
    groups, cams, deg = scene_render.object_layout(dev) if name == "object" else scene_render.scene_layout(dev)
    bg = torch.zeros(3, device=dev)
    S_of = lambda it: scene_render.settings(cams(it)[:1], deg, bg)
    gt = torch.rand(G, 3, 512, 512, device=dev, generator=torch.Generator(device=dev).manual_seed(0)).half()
    variants = {"eager": Eager(clone(groups), gt), "graph": Graph(clone(groups), gt, False),
                "target": Graph(clone(groups), gt, True)}
    P = sum(int(g["_xyz"].shape[0]) for g in groups)
    del groups
    res = {k: {"sync_ms": [], "b2b_ms": [], "host_us": []} for k in variants}
    variants["eager"].step(S_of(0), 0)  # one-time library / allocator initialisation, untimed
    torch.cuda.synchronize()
    capture = {}
    for k in ("graph", "target"):
        t0 = time.perf_counter()
        variants[k].step(S_of(1), 1)    # measurement + capture + first replay
        torch.cuda.synchronize()
        capture[k] = round((time.perf_counter() - t0) * 1e3, 2)
    it = 2
    for _ in range(args.warmup):
        for v in variants.values():
            v.step(S_of(it), it)
            it += 1
    for k in ("graph", "target"):
        variants[k].sg.check()
    settings = [S_of(j) for j in range(args.steps)]
    for _ in range(args.rounds):
        for k, v in variants.items():            # alternate the variants
            for j in range(args.steps):
                torch.cuda.synchronize()
                t0 = time.perf_counter()
                v.step(settings[j], it + j)
                torch.cuda.synchronize()
                res[k]["sync_ms"].append((time.perf_counter() - t0) * 1e3)
            torch.cuda.synchronize()
            t0 = time.perf_counter()
            for j in range(args.steps):
                v.step(settings[j], it + j)
            t1 = time.perf_counter()
            torch.cuda.synchronize()
            t2 = time.perf_counter()
            res[k]["b2b_ms"].append((t2 - t0) * 1e3 / args.steps)
            res[k]["host_us"].append((t1 - t0) * 1e6 / args.steps)
            it += args.steps
    for k in ("graph", "target"):
        variants[k].sg.check()
    out = {"layout": name, "views": 1, "size": 512, "P": P}
    med = lambda xs: round(sorted(xs)[len(xs) // 2], 4)
    for k, v in variants.items():
        r = res[k]
        dev_ms, loss_ms = device_ms(lambda: v.step(settings[0], it), 10)
        out[k] = {"sync_ms": med(r["sync_ms"]), "b2b_ms": med(r["b2b_ms"]), "b2b_ms_range": [round(min(r["b2b_ms"]), 4),
                  round(max(r["b2b_ms"]), 4)], "host_us": round(med(r["host_us"]), 1), "device_ms": dev_ms}
        if k == "target":
            out[k]["recon_l2_ms"] = loss_ms
        if k in capture:
            out[k]["capture_ms"] = capture[k]
    return out


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--steps", type=int, default=20)
    ap.add_argument("--warmup", type=int, default=3)
    ap.add_argument("--rounds", type=int, default=3)
    ap.add_argument("--layouts", default="object,scene")
    a = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("recon_step.py measures on the GPU; no CUDA device found")
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
