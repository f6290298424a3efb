#!/usr/bin/env python
"""What bounded the multisplit key scatter when it wrote one 8-byte store per pair (the binning before the padded key
buffer of csrc/binning.cu)?

Runs one library forward of a bench.py workload with a caller-owned scratch buffer, takes the scatter's real inputs
from it (rectdepth, the per-CTA tile histograms ms_hist, the tile starts the scan wrote) and times four kernels of
benchmarks/scatter_probe.cu on them with CUDA events, alternated launch by launch:

  scatter      those statements: every pair is one 8-byte store to its slot of the CTA's tile slice
  l2_sink      the same instructions and atomics, each key stored to dummy[pos & mask] (a 4 MB buffer that stays in L2)
  no_store     the same loop and atomics without the store
  stream       a coalesced write of the same number of keys (the output's byte floor)

If l2_sink is far below scatter, the scatter is bound by where its stores land (partly written 32-byte sectors
evicted from L2 to HBM), not by the loop or the atomics.  The scatter kernel's output is checked against the
library's sorted key lists.  The measured table is in BASELINE.md §3.  The probe compiles scatter_probe.cu with nvcc into a temporary directory.

  python benchmarks/scatter_probe.py [--workloads cfg3_1M_1024,cfg3b_1M_1024_screenfill] [--iters 200] [--out FILE]
"""
import argparse
import ctypes as C
import json
import os
import subprocess
import sys
import tempfile

import numpy as np
import torch

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(HERE)
sys.path.insert(0, ROOT)
import bench  # noqa: E402
from dreamscene_b200 import GaussianRasterizationSettings, _build, _lib  # noqa: E402
from dreamscene_b200 import rasterizer as R  # noqa: E402

VARIANTS = ("scatter", "l2_sink", "no_store", "stream")
MS_ITEMS, MS_WAVE_CTAS = 4, 264


def ms_blocks(P):
    """gsr_ms_blocks of csrc/common.cuh."""
    full = (P + 1024 * MS_ITEMS - 1) // (1024 * MS_ITEMS)
    if full >= MS_WAVE_CTAS:
        return full
    return max(1, min((P + 255) // 256, MS_WAVE_CTAS))


def build_probe(tmp):
    so = os.path.join(tmp, "scatter_probe.so")
    cmd = [_build._nvcc(), "-gencode", "arch=compute_90a,code=sm_90a", "-O3", "-std=c++17", "-shared",
           "-Xcompiler", "-fPIC", os.path.join(HERE, "scatter_probe.cu"), "-o", so]
    subprocess.run(cmd, check=True)
    lib = C.CDLL(so)
    lib.probe_launch.restype = C.c_int
    lib.probe_launch.argtypes = [C.c_int] * 6 + [C.c_uint32] + [C.c_void_p] * 5 + [C.c_uint32, C.c_uint64, C.c_void_p]
    return lib


def scatter_inputs(name, dev):
    """One library forward of workload `name` -> the scatter's inputs and the sorted key lists."""
    wl = bench.WORKLOADS[name]
    sc, cam, _, _ = bench.make_scene(wl, 0)
    P, H, W = wl["P"], wl["H"], wl["W"]
    t = {k: sc[k].to(dev).contiguous() for k in ("means3D", "opacities", "shs", "scales", "rotations")}
    S = GaussianRasterizationSettings(
        image_height=H, image_width=W, tanfovx=cam.tanfovx, tanfovy=cam.tanfovy, bg=torch.ones(3, device=dev),
        scale_modifier=1.0, viewmatrix=cam.world_view_transform.to(dev), projmatrix=cam.full_proj_transform.to(dev),
        sh_degree=3, campos=cam.camera_center.to(dev), prefiltered=False, score_flag=False)
    keep = []
    prm = R._make_params(S, P, 16, keep, dev, S.bg.contiguous())
    lib = _lib.load()
    cap = 32 << 20
    sl, vl = _lib.scratch_layout(P, H, W, cap), _lib.saved_layout(P, H, W, cap, False)
    scratch = torch.zeros(sl.total, dtype=torch.uint8, device=dev)
    saved = torch.zeros(vl.total, dtype=torch.uint8, device=dev)
    color = torch.empty(3, H, W, device=dev)
    da = torch.empty(2, H, W, device=dev)
    radii = torch.empty(P, dtype=torch.int32, device=dev)
    p = _lib.ptr
    _lib.check(lib.b200gsr_forward(C.byref(prm), p(t["means3D"]), p(t["shs"]), None, p(t["opacities"]), p(t["scales"]),
                                   p(t["rotations"]), None, p(color), p(da), p(radii), None, p(scratch), sl.total,
                                   p(saved), vl.total, cap, _lib.FWD_NO_BACKWARD, None, 0, _lib.stream(dev)),
               "b200gsr_forward")
    torch.cuda.synchronize(dev)
    gx, gy = (W + 15) // 16, (H + 15) // 16
    ntiles = gx * gy
    D = int(saved[vl.header:vl.header + 4].view(torch.int32).item())
    assert D <= cap
    nblk = ms_blocks(P)
    return dict(P=P, D=D, gx=gx, ntiles=ntiles, nblk=nblk, per=(P + nblk - 1) // nblk, cap=cap,
                rectdepth=scratch[sl.rectdepth:sl.rectdepth + 16 * P].clone(),
                ms_hist=scratch[sl.ms_hist:sl.ms_hist + 4 * nblk * ntiles].clone(),
                tile_start=saved[vl.tile_start:vl.tile_start + 4 * (ntiles + 1)].view(torch.int32).clone(),
                keys_sorted=saved[vl.keys:vl.keys + 8 * D].view(torch.int64).clone())


def check_scatter(x, keys):
    """The probe's scatter wrote, per tile, the same keys as the library's (sorted) lists."""
    D = x["D"]
    k = keys[:D]
    order = torch.sort(k, stable=True).indices      # depth bits are a non-negative float's: int64 order is key order
    tile = torch.searchsorted(x["tile_start"][1:].long(), order, right=True)   # tile of each slot, in key order
    order = order[torch.sort(tile, stable=True).indices]
    return bool(torch.equal(k[order], x["keys_sorted"]))


def run(lib, x, iters, dev):
    D = x["D"]
    keys = torch.empty(x["cap"], dtype=torch.int64, device=dev)
    dummy = torch.empty(1 << 19, dtype=torch.int64, device=dev)          # 4 MB
    cursor = torch.empty(x["ntiles"], dtype=torch.int32, device=dev)
    st = _lib.stream(dev)

    def launch(mode):
        cursor.copy_(x["tile_start"][:x["ntiles"]])
        rc = lib.probe_launch(mode, x["P"], x["nblk"], x["per"], x["gx"], x["ntiles"], x["cap"],
                              x["rectdepth"].data_ptr(), cursor.data_ptr(), x["ms_hist"].data_ptr(), keys.data_ptr(),
                              dummy.data_ptr(), (1 << 19) - 1, D, st)
        assert rc == 0, rc

    launch(0)
    torch.cuda.synchronize(dev)
    ok = check_scatter(x, keys)
    for m in range(4):
        for _ in range(5):
            launch(m)
    ev = [[(torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)) for _ in range(iters)]
          for _ in VARIANTS]
    for i in range(iters):
        for m in range(4):
            m = (m + i) % 4
            cursor.copy_(x["tile_start"][:x["ntiles"]])
            ev[m][i][0].record()
            launch(m)
            ev[m][i][1].record()
    torch.cuda.synchronize(dev)
    out = {}
    for m, name in enumerate(VARIANTS):
        t = np.array([a.elapsed_time(b) for a, b in ev[m]])
        out[name] = {"median_ms": float(np.median(t)), "p10_ms": float(np.percentile(t, 10)),
                     "p90_ms": float(np.percentile(t, 90))}
    return ok, out


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--workloads", default="cfg3_1M_1024,cfg3b_1M_1024_screenfill")
    ap.add_argument("--iters", type=int, default=200)
    ap.add_argument("--out", default=None, help="also write the results as JSON to this file")
    args = ap.parse_args()
    assert torch.cuda.is_available(), "the probe needs a CUDA device"
    dev = torch.device("cuda", 0)
    torch.cuda.set_device(dev)
    q = subprocess.run(["nvidia-smi", "-i", "0", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                       capture_output=True, text=True).stdout.strip()
    props = torch.cuda.get_device_properties(dev)
    res = {"gpu": q or props.name, "l2_bytes": getattr(props, "L2_cache_size", None), "workloads": {}}
    with tempfile.TemporaryDirectory() as tmp:
        lib = build_probe(tmp)
        for name in args.workloads.split(","):
            x = scatter_inputs(name, dev)
            ok, t = run(lib, x, args.iters, dev)
            res["workloads"][name] = {"tile_pairs": x["D"], "key_mb": x["D"] * 8 / 1e6, "ctas": x["nblk"],
                                      "tiles": x["ntiles"], "scatter_matches_library": ok, "times": t}
            print(f"{name}: D={x['D']} ({x['D'] * 8 / 1e6:.1f} MB of keys), {x['nblk']} CTAs, "
                  f"scatter output matches the library's lists: {ok}")
            for v in VARIANTS:
                print(f"  {v:9s} median {t[v]['median_ms']:.4f} ms  (p10 {t[v]['p10_ms']:.4f}, p90 {t[v]['p90_ms']:.4f})")
    print(f"GPU: {res['gpu']}, L2 {res['l2_bytes']} B")
    if args.out:
        with open(args.out, "w") as f:
            json.dump(res, f, indent=1)


if __name__ == "__main__":
    main()
