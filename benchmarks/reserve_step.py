#!/usr/bin/env python
"""Reserved-row groups (DESIGN.md f13) against plain groups that re-capture the replayed step after every event.

Object layout (benchmarks/scene_render.py: 1.2 M Gaussians, M = 16, sh_degree 3), 4 views of 512 x 512, one group.
1. schedule: `steps` replayed steps with statistics, and every `every` steps the reference's densify step
   (step(optimize=False)) followed by a densify_and_prune (max_grad = the 0.9 quantile of the statistics' mean
   gradient, so each event adds roughly a tenth of the rows).  Variants, alternating in rounds:
     plain    : densify.densify_and_prune, then new leaves, a new GaussianAdam state and new statistics handed to the
                StepGraph, which captures again at the next render (INTEGRATION.md section 4b)
     reserved : ReservedGroup(capacity = 2 x the start count).densify_and_prune in place; the graphs replay
   Reported: total wall time of the schedule, and each event's cost = the event plus the first step after it.
2. steady state: ms/step of back-to-back replayed steps at the same live count with 0 % (plain group), 50 % and
   100 % headroom, alternating: the price of the dead rows.
Prints one JSON line with the card's name, power limit and max SM clock read in the same run.

  python benchmarks/reserve_step.py [--steps 60] [--every 20] [--rounds 3] [--steady-steps 20]
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
from dreamscene_b200 import densify as D  # noqa: E402
from dreamscene_b200.reserve import ReservedGroup  # noqa: E402
import scene_render  # noqa: E402

NAMES = scene_render.NAMES
LRS = {"_xyz": 1.6e-4, "_opacity": 0.05, "_scaling": 0.005, "_rotation": 0.001, "_features_dc": 0.0025,
       "_features_rest": 0.000125}
DNAME = {"xyz": "_xyz", "f_dc": "_features_dc", "f_rest": "_features_rest", "opacity": "_opacity",
         "scaling": "_scaling", "rotation": "_rotation"}


def _opt(g):
    get = (lambda k: g[k]) if isinstance(g, dict) else (lambda k: getattr(g, k))
    return GaussianAdam([{"params": [get(k)], "lr": LRS[k]} for k in NAMES], lr=0.0, eps=1e-15)


class Plain:
    """One plain group: every event builds new leaves, optimizer state and statistics (the StepGraph re-captures)."""
    def __init__(self, g, dev):
        self.dev = dev
        self._set({k: v.detach().clone() for k, v in g.items()}, None)

    def _set(self, leaves, moments, step=None):
        self.g = {k: v.requires_grad_(True) for k, v in leaves.items()}
        self.opt = _opt(self.g)
        if moments is not None:
            for dk, (m, v) in moments.items():
                self.opt.state[self.g[DNAME[dk]]] = {"step": step.clone(), "exp_avg": m, "exp_avg_sq": v}
        n = int(self.g["_xyz"].shape[0])
        self.stats = (torch.zeros(n, 1, device=self.dev), torch.zeros(n, 1, device=self.dev),
                      torch.zeros(n, device=self.dev))
        if hasattr(self, "sg"):
            self.sg.groups, self.sg.optimizers, self.sg.densify_stats = [self.g], [self.opt], [self.stats]
        else:
            self.sg = StepGraph([self.g], [self.opt], views=4, height=512, width=512, densify_stats=[self.stats],
                                keep_means2D=False)

    @property
    def live(self):
        return int(self.g["_xyz"].shape[0])

    def densify(self, max_grad, seed):
        params = {dk: self.g[k].detach() for dk, k in DNAME.items()}
        st = self.opt.state[self.g["_xyz"]]
        adam = {dk: (self.opt.state[self.g[k]]["exp_avg"], self.opt.state[self.g[k]]["exp_avg_sq"])
                for dk, k in DNAME.items()}
        new_p, new_a, _ = D.densify_and_prune(params, adam, self.stats[0], self.stats[1], max_grad, 0.005, 5.0, None,
                                              generator=torch.Generator(device=self.dev).manual_seed(seed))
        self._set({k: new_p[dk] for dk, k in DNAME.items()}, new_a, st["step"])


class Reserved:
    def __init__(self, g, dev, headroom=1.0):
        self.g = ReservedGroup.from_tensors(g["_xyz"], g["_features_dc"], g["_features_rest"], g["_opacity"],
                                            g["_scaling"], g["_rotation"], headroom=headroom)
        self.opt = _opt(self.g)
        self.dev = dev
        self.sg = StepGraph([self.g], [self.opt], views=4, height=512, width=512, densify_stats=[self.g],
                            keep_means2D=False)
        self.stats = self.g.stats

    @property
    def live(self):
        return self.g.live_count

    def densify(self, max_grad, seed):
        self.g.densify_and_prune(self.opt, max_grad, 0.005, 5.0, None,
                                 generator=torch.Generator(device=self.dev).manual_seed(seed))


def step(v, S, it, target, optimize=True):
    flags = [(k + it) % 2 == 0 for k in range(len(S))]
    out = v.sg.render(S, shs_aug=flags, scale_aug=flags, seed=it)
    (((out.image - target) ** 2).mean() + 0.01 * out.disp.mean()).backward()
    v.sg.step(optimize=optimize, stats_view=-1)


def max_grad(v):
    n = v.live
    g = (v.stats[0].view(-1)[:n] / v.stats[1].view(-1)[:n]).nan_to_num(0.0)
    return float(torch.quantile(g[torch.randperm(n, device=g.device)[:1 << 20]], 0.9))


def schedule(v, args, S_of, target):
    """-> (total ms, [event + first step ms])."""
    events = []
    torch.cuda.synchronize()
    t0 = time.perf_counter()
    for it in range(1, args.steps + 1):
        if it % args.every == 0:
            step(v, S_of(it), it, target, optimize=False)
            torch.cuda.synchronize()
            te = time.perf_counter()
            v.densify(max_grad(v), it)
            step(v, S_of(it + 1), it + 1, target)
            torch.cuda.synchronize()
            events.append(round((time.perf_counter() - te) * 1e3, 2))
        else:
            step(v, S_of(it), it, target)
    torch.cuda.synchronize()
    return round((time.perf_counter() - t0) * 1e3, 1), events


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--steps", type=int, default=60)
    ap.add_argument("--every", type=int, default=20)
    ap.add_argument("--rounds", type=int, default=3)
    ap.add_argument("--steady-steps", type=int, default=20)
    a = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("reserve_step.py measures on the GPU; no CUDA device found")
    dev = torch.device("cuda", 0)
    torch.manual_seed(0)
    info = scene_render.gpu_info()
    groups, cams, deg = scene_render.object_layout(dev)
    g0 = {k: v.detach() for k, v in groups[0].items()}
    bg = torch.zeros(3, device=dev)
    S_of = lambda it: scene_render.settings(cams(it), deg, bg)
    target = torch.rand(4, 3, 512, 512, device=dev, generator=torch.Generator(device=dev).manual_seed(0))
    out = {"layout": "object", "views": 4, "size": 512, "P": int(g0["_xyz"].shape[0]), "every": a.every,
           "steps": a.steps, "gpu": info}
    # 1. the schedule, plain and reserved alternating, fresh groups each round (the first round warms everything up)
    res = {"plain": [], "reserved": []}
    for r in range(a.rounds + 1):
        for name, cls in (("plain", Plain), ("reserved", Reserved)):
            v = cls(g0, dev)
            step(v, S_of(0), 0, target)
            total, events = schedule(v, a, S_of, target)
            v.sg.check()
            if r:
                res[name].append({"total_ms": total, "event_ms": events, "live_end": v.live})
            del v
            torch.cuda.empty_cache()
    out["schedule"] = res
    # 2. steady state at the start count with 0 %, 50 % and 100 % headroom
    variants = {"0%": Plain(g0, dev), "50%": Reserved(g0, dev, 0.5), "100%": Reserved(g0, dev, 1.0)}
    for v in variants.values():
        for j in range(3):
            step(v, S_of(j), j, target)
    settings = [S_of(j) for j in range(a.steady_steps)]
    times = {k: [] for k in variants}
    for _ in range(5):
        for k, v in variants.items():
            torch.cuda.synchronize()
            t0 = time.perf_counter()
            for j in range(a.steady_steps):
                step(v, settings[j], 100 + j, target)
            torch.cuda.synchronize()
            times[k].append((time.perf_counter() - t0) * 1e3 / a.steady_steps)
    for v in variants.values():
        v.sg.check()
    out["steady_ms_per_step"] = {k: {"median": round(sorted(t)[len(t) // 2], 4),
                                     "range": [round(min(t), 4), round(max(t), 4)]} for k, t in times.items()}
    print(json.dumps(out), flush=True)


if __name__ == "__main__":
    main()
