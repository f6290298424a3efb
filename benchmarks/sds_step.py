#!/usr/bin/env python
"""The guidance stages' step: eager, StepGraph with the regularisers eager, and StepGraph with the regularisers inside
its graphs (DESIGN.md f10).

  eager : render_scene(groups, S, return_scales=True) + disparity_from_depth_alpha + loss + backward
          + GaussianAdam.step() per group
  graph : sg.render(S) + the same loss + backward + sg.step()
  reg   : StepGraph(..., tv_weight=, tv_depth_weight=, scale_weight=): sg.render(S) + the guidance term alone
          + backward + sg.step()

The loss is the reference's (object_trainer.py:378-381, scene_trainer.py:867-877), with an L2 against a fixed target
standing in for the guidance term and written first:

    l2(image, target) + lambda_tv * tv_loss(image) + lambda_tv_depth * tv_loss(disp) + lambda_scale * scale_loss(scales)

tv_loss and scale_loss (mean(mean(scales, -1))) are the restated reference expressions (harness/regularisers_ref.py).  The weights are the reference's:
lambda_tv 1, lambda_tv_depth 1 (object) / 0 (scene), lambda_scale 1 (object) / 0.5 (scene).  The eager variants keep a
term of weight 0 (the reference computes 0 * tv_loss(depths)); reg leaves it out.  Every step changes the cameras,
flags, seed and xyz lr.  Layouts as benchmarks/step_graph.py:
  object : 1.2 M Gaussians in one group, M = 16, 4 views of 512 x 512
  scene  : harness/room.py::build_scene (cfg5: 2.63 M Gaussians in 6 groups, M = 4), 4 views of 512 x 512

Per variant, alternating the variants in rounds:
  sync_ms    : median wall time of one step followed by torch.cuda.synchronize()
  b2b_ms     : wall time per step of `steps` back-to-back steps with one synchronize at the end (median, range)
  host_us    : host time per step in the back-to-back run (until the last call returns, before the synchronize)
  device_ms  : summed CUDA kernel and copy time per step from torch.profiler, after the timed rounds and apart from
               them; for reg also the new tv_loss / scale_loss kernels' share (reg_kernels_ms)
  capture_ms : the graph's first step (eager measurement + capture + the first replay), timed after one eager step
               has initialised the library and the allocator
Prints one JSON line per layout, with the card's name, power limit and max SM clock read in the same run.

  python benchmarks/sds_step.py [--steps 20] [--rounds 5] [--layouts object,scene]
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
from harness.regularisers_ref import scale_loss, tv_loss  # noqa: E402
import scene_render  # noqa: E402

NAMES = scene_render.NAMES
LRS = {"_xyz": 1.6e-4, "_opacity": 0.05, "_scaling": 0.005, "_rotation": 0.001, "_features_dc": 0.0025,
       "_features_rest": 0.000125}
WEIGHTS = {"object": (1.0, 1.0, 1.0), "scene": (1.0, 0.0, 0.5)}     # lambda_tv, lambda_tv_depth, lambda_scale


def clone(groups):
    return [{k: v.detach().clone().requires_grad_(True) for k, v in g.items()} for g in groups]


def optimizers(groups):
    return [GaussianAdam([{"params": [g[k]], "lr": LRS[k]} for k in NAMES], lr=0.0, eps=1e-15) for g in groups]


def guidance(image, target):
    return ((image - target) ** 2).mean()


def full_loss(image, disp, scales, target, w):
    return guidance(image, target) + w[0] * tv_loss(image) + w[1] * tv_loss(disp) + w[2] * scale_loss(scales)


def flags_of(B, it):
    return [(v + it) % 2 == 0 for v in range(B)]


class Eager:
    def __init__(self, groups, w):
        self.groups, self.opts, self.w = groups, optimizers(groups), w

    def step(self, S, it, target):
        for o in self.opts:
            o.param_groups[0]["lr"] = LRS["_xyz"] * 0.99 ** it
        flags = flags_of(len(S), it)
        outs, scales = render_scene(self.groups, S, shs_aug=flags, scale_aug=flags, seed=it, return_scales=True)
        image = torch.stack([o[0] for o in outs])
        disp, _ = disparity_from_depth_alpha(torch.stack([o[2] for o in outs]),
                                             [1.0 / (2.0 * float(s.tanfovx)) for s in S])
        full_loss(image, disp, scales, target, self.w).backward()
        for o in self.opts:
            o.step()
            o.zero_grad()


class Graph:
    def __init__(self, groups, B, w, reg):
        self.groups, self.opts, self.w, self.reg = groups, optimizers(groups), w, reg
        kw = dict(tv_weight=w[0], tv_depth_weight=w[1], scale_weight=w[2]) if reg else {}
        self.sg = StepGraph(groups, self.opts, views=B, height=512, width=512, **kw)

    def step(self, S, it, target):
        for o in self.opts:
            o.param_groups[0]["lr"] = LRS["_xyz"] * 0.99 ** it
        flags = flags_of(len(S), it)
        out = self.sg.render(S, shs_aug=flags, scale_aug=flags, seed=it)
        if self.reg:
            guidance(out.image, target).backward()
        else:
            full_loss(out.image, out.disp, out.scales, target, self.w).backward()
        self.sg.step()


def device_ms(run, steps):
    """-> (all kernels and copies, the tv_loss / scale_loss kernels) in ms per step."""
    from torch.autograd import DeviceType
    with torch.profiler.profile(activities=[torch.profiler.ProfilerActivity.CUDA]) as prof:
        for _ in range(steps):
            run()
        torch.cuda.synchronize()
    ev = [e for e in prof.events() if e.device_type == DeviceType.CUDA]
    tot = lambda pred: round(sum(e.self_device_time_total for e in ev if pred(e.name)) / 1e3 / steps, 4)
    ours = ("tv_kernel", "tv_finish_kernel", "scale_loss_kernel", "scale_finish_kernel")
    return tot(lambda n: True), tot(lambda n: any(k in n for k in ours))


def run_layout(name, args, dev):
    groups, cams, deg = scene_render.object_layout(dev) if name == "object" else scene_render.scene_layout(dev)
    bg = torch.zeros(3, device=dev)
    S_of = lambda it: scene_render.settings(cams(it), deg, bg)
    target = torch.rand(4, 3, 512, 512, device=dev, generator=torch.Generator(device=dev).manual_seed(0))
    w = WEIGHTS[name]
    variants = {"eager": Eager(clone(groups), w), "graph": Graph(clone(groups), 4, w, False),
                "reg": Graph(clone(groups), 4, w, True)}
    P = sum(int(g["_xyz"].shape[0]) for g in groups)
    del groups
    res = {k: {"sync_ms": [], "b2b_ms": [], "host_us": []} for k in variants}
    variants["eager"].step(S_of(0), 0, target)  # one-time library / allocator initialisation, untimed
    torch.cuda.synchronize()
    capture = {}
    for k in ("graph", "reg"):
        t0 = time.perf_counter()
        variants[k].step(S_of(1), 1, target)    # measurement + capture + first replay
        torch.cuda.synchronize()
        capture[k] = round((time.perf_counter() - t0) * 1e3, 2)
    it = 2
    for _ in range(args.warmup):
        for v in variants.values():
            v.step(S_of(it), it, target)
            it += 1
    for k in ("graph", "reg"):
        variants[k].sg.check()
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
    for k in ("graph", "reg"):
        variants[k].sg.check()
    out = {"layout": name, "views": 4, "size": 512, "P": P, "weights": list(w)}
    med = lambda xs: round(sorted(xs)[len(xs) // 2], 4)
    for k, v in variants.items():
        r = res[k]
        dev_ms, reg_ms = device_ms(lambda: v.step(settings[0], it, target), 5)
        out[k] = {"sync_ms": med(r["sync_ms"]), "b2b_ms": med(r["b2b_ms"]), "b2b_ms_range": [round(min(r["b2b_ms"]), 4),
                  round(max(r["b2b_ms"]), 4)], "host_us": round(med(r["host_us"]), 1), "device_ms": dev_ms}
        if k == "reg":
            out[k]["reg_kernels_ms"] = reg_ms
        if k in capture:
            out[k]["capture_ms"] = capture[k]
    return out


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--steps", type=int, default=20)
    ap.add_argument("--warmup", type=int, default=3)
    ap.add_argument("--rounds", type=int, default=5)
    ap.add_argument("--layouts", default="object,scene")
    a = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("sds_step.py measures on the GPU; no CUDA device found")
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
