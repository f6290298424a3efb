"""The rasterizer against the oracle from inside the room DreamScene's scene stages render (harness/room.py, the cfg5
scene): most Gaussians behind the camera or just past the 0.2 near plane, thousands outside the 1.3 tanfov EWA clamp,
tile rectangles clipped on every side, footprints covering the whole image.  The ball scenes of the other parity
tests, seen from outside, reach none of these branches.

Yardsticks as everywhere: integers (radii, tile ranges, sorted ids, depth bits) bit-exact, the forward through
parity_budgets.check_forward, every gradient norm-wise within BWD_REL of the fp64 oracle evaluated on the fp32 run's
decisions: pair lists, blend decisions and the EWA / colour clamp flags."""
import math

import numpy as np
import pytest
import torch

from harness import room
from oracle import splat_ref as O
from tests import parity_budgets as B
from tests import parity_tools as PT
from tests import room_edges as E
from tests import util_scene as U
from tests.test_gpu_parity import check_lists, run_cuda, run_oracle

pytestmark = pytest.mark.gpu

DEG, M = 1, 4
SMALL = dict(n_wall=6000, n_floor=7800, n_obj=3000, scale_mul=16.0)     # 49 800 Gaussians, about as opaque as cfg5
GRADS = ("means3D", "scales", "rotations", "opacities", "shs", "means2D")


def small_room():
    return room.rasterizer_inputs(room.build_scene("cpu", M=M, **SMALL))


def wall_camera(size):
    """0.3 m in front of the room's +x wall, looking at it."""
    return room.look_camera([room.ROOM[0] / 2 - 0.3, 0.4, 1.3], [1.0, 0.0, 0.0], size, "cpu")


def views(size):
    return [room.scene_camera(k, size, "cpu") for k in range(3)] + [wall_camera(size)]


def incoming(H, W, seed):
    g = torch.Generator().manual_seed(seed)
    return torch.randn(3, H, W, generator=g) / (H * W), torch.randn(2, H, W, generator=g) / (H * W)


def branch_census(pre, H, W):
    """How much of the edge geometry a view holds."""
    vis = pre["visible"].numpy()
    px, py = pre["px"].detach().numpy(), pre["py"].detach().numpy()
    r = pre["radii"].numpy().astype(np.float64)
    gx, gy = (W + 15) // 16, (H + 15) // 16
    clipped = vis & ((px - r < 0) | (py - r < 0) | (px + r + 15 >= 16 * (gx + 1)) | (py + r + 15 >= 16 * (gy + 1)))
    rect = pre["rect"].numpy()
    return dict(near=float((pre["depth"].detach() <= O.NEAR_Z).float().mean()),
                out_x=int((vis & ~pre["in_x"].numpy()).sum()), out_y=int((vis & ~pre["in_y"].numpy()).sum()),
                clipped=int(clipped.sum()),
                whole=int((vis & (rect[:, 0] == 0) & (rect[:, 1] == 0) & (rect[:, 2] == gx) & (rect[:, 3] == gy)).sum()))


def full_frame(sc, cam, config, seed, kernel_clamps=()):
    """CUDA vs oracle on the whole frame: lists, forward, n_contrib, all six gradients (fp64 on the fp32 decisions).
    kernel_clamps: rows whose colour the oracle's fp32 puts at exactly 0 and the kernels' fused multiply-adds just
    below it (DESIGN.md section 8 item 8): the oracle is evaluated on the kernels' clamp decision for them, and the
    kernels' SH gradient of those rows must be exactly zero."""
    H, W = cam.image_height, cam.image_width
    gc, gd = incoming(H, W, seed)
    ref32 = run_oracle(sc, cam, DEG, record=True)
    rows = list(kernel_clamps)
    if rows:
        pre = ref32["pre"]
        assert not bool(pre["clamped"][rows].any()) and bool((pre["rgb"][rows] == 0).all())
        ref32["decisions"]["clamped"] = pre["clamped"].clone()
        ref32["decisions"]["clamped"][rows] = True
    cu = run_cuda(sc, cam, DEG, grads=(gc, gd))
    np.testing.assert_array_equal(cu["radii"].cpu().numpy(), ref32["radii"].numpy())
    dec = check_lists(sc, cam, ref32)
    stats = PT.forward_stats(cu["color"], cu["depth_alpha"], ref32["color"], ref32["depth_alpha"],
                             cu_nc=dec["n_contrib"], ref_nc=ref32["n_contrib"].numpy())
    B.check_forward(config, stats)
    tiles = [t for t in range(len(ref32["ranges"])) if ref32["ranges"][t, 1] > ref32["ranges"][t, 0]]
    want = PT.oracle_backward_on_tiles(sc, cam, DEG, tiles, gc, gd, ref32["decisions"],
                                       blend=ref32["decisions"]["blend"])
    if rows:
        assert float(cu["grads"]["shs"][rows].abs().max()) == 0.0
        assert float(want["shs"][rows].abs().max()) == 0.0
    errs = PT.grad_errors(cu["grads"], want)
    print(config, {k: stats[k]["max_abs"] for k in ("color", "depth", "T")}, stats["n_contrib"]["n_mismatch"],
          {k: errs[k]["rel_l2"] for k in GRADS})
    for k in GRADS:
        assert errs[k]["rel_l2"] < B.BWD_REL, (k, errs[k])
    return ref32, cu, want, dec


@pytest.mark.parametrize("size", [200, 256])        # 200: a partial last tile row and column
def test_small_room_full_frame_matches_the_oracle(size):
    sc = small_room()
    census = []
    for v, cam in enumerate(views(size)):
        ref32, _, _, _ = full_frame(sc, cam, "room_small", seed=10 * v + size)
        c = branch_census(ref32["pre"], size, size)
        n = ref32["ranges"][:, 1] - ref32["ranges"][:, 0]
        assert (n > 0).all(), "every tile of a view from inside the room holds Gaussians"
        census.append(c)
    print("census", size, census)
    # the scene really reaches the branches (a later change to it must not empty this test)
    assert all(c["near"] > 0.3 for c in census)
    assert sum(c["out_x"] for c in census) > 200 and sum(c["out_y"] for c in census) > 200
    assert all(c["clipped"] > 100 for c in census)
    assert sum(c["whole"] for c in census) >= 1


def _edge_scene(rows_fn, size=192):
    cam = E.axis_camera(size)
    E.check_axis_camera(cam)
    rows = rows_fn(cam, np.random.RandomState(7))
    sc0 = small_room()
    sc = E.append(sc0, E.as_inputs(rows, M))
    return cam, rows, sc, sc0["means3D"].shape[0]


def test_constructed_edge_gaussians_match_the_oracle():
    """Near plane to the ulp, clamp limits to the ulp, footprints containing the camera, behind it, clipped on every
    side and corner, centres far off-screen, colours an ulp either side of the clamp, all inside the small room."""
    from oracle import fp32_arbiter as A
    cam, rows, sc, P0 = _edge_scene(E.edge_rows)
    H = W = cam.image_width
    kinds = np.array([r["kind"] for r in rows])
    idx = np.arange(P0, P0 + len(rows))
    ref32, cu, want, dec = full_frame(sc, cam, "room_small", seed=99, kernel_clamps=idx[kinds == "colour0_exact"])
    pre = ref32["pre"]
    # the constructed rows on their own (each ratio group holds the rows exactly at +-limit): a branch taken on the
    # wrong side of a boundary moves a handful of rows, which the norm over the whole room would not show
    for group in ("ratio_x", "ratio_y", None):
        sel = idx if group is None else idx[kinds == group]
        for k in GRADS:
            e = U.rel_err(cu["grads"][k][sel], want[k][sel])
            print("edge rows", group, k, e)
            assert e < B.BWD_REL, (group, k, e)
    # the constructions are what they claim, read back through the oracle's fp32 chain
    tz = pre["depth"].detach().numpy()[idx]
    near = idx[kinds == "near"] - P0
    np.testing.assert_array_equal(tz[near].view(np.uint32).astype(np.int64) - int(np.float32(0.2).view(np.uint32)),
                                  [-2, -1, 0, 1, 2])
    np.testing.assert_array_equal(pre["visible"].numpy()[idx][near], [False, False, False, True, True])
    assert not pre["visible"].numpy()[idx][kinds == "behind"].any()
    assert pre["visible"].numpy()[idx][kinds == "clipped"].all()
    in_x, in_y = pre["in_x"].numpy()[idx], pre["in_y"].numpy()[idx]
    np.testing.assert_array_equal(in_x[kinds == "ratio_x"], [True, True, False, False, True, True])
    np.testing.assert_array_equal(in_y[kinds == "ratio_y"], [True, True, False, False, True, True])
    assert pre["visible"].numpy()[idx][np.isin(kinds, ["ratio_x", "ratio_y"])].all()
    # cull decision, radius and tile rectangle bit-exact for every constructed Gaussian: CUDA's rect read back from its
    # sorted list, the oracle's and a third fp32 evaluation (the numpy scalar arbiter)
    gx = (W + 15) // 16
    ts = dec["tile_start"]
    tile_of = np.repeat(np.arange(len(ts) - 1), np.diff(ts))
    radii = cu["radii"].cpu().numpy()
    V, F = cam.world_view_transform.numpy(), cam.full_proj_transform.numpy()
    for i in idx:
        arb = A.radius_rect(sc["means3D"][i].numpy(), sc["scales"][i].numpy(), sc["rotations"][i].numpy(), V, F,
                            cam.tanfovx, cam.tanfovy, H, W)
        assert arb["visible"] == bool(radii[i] > 0) and arb["radius"] == radii[i], (i, kinds[i - P0], arb)
        t = tile_of[dec["idx"] == i]
        if arb["visible"]:
            got = (int((t % gx).min()), int((t // gx).min()), int((t % gx).max()) + 1, int((t // gx).max()) + 1)
            assert got == tuple(arb["rect"]) == tuple(pre["rect"][i].tolist()), (i, kinds[i - P0], got, arb["rect"])
            assert len(t) == (got[2] - got[0]) * (got[3] - got[1])
        else:
            assert t.size == 0


def test_near_singular_footprints_match_the_oracle():
    """Large flat Gaussians edge-on at t.z ~ 0.25 (a c / det ~ 300, det = a c - b^2 cancels about 8 of its bits), as the
    room's wall and floor splats are when seen edge-on near the camera: the whole frame against the oracle as
    everywhere, and the near-singular rows on their own against fp64 within BWD_REL."""
    cam, rows, sc, P0 = _edge_scene(E.near_singular_rows)
    a, b, c = (x.detach().numpy()[P0:] for x in O.preprocess(U.oracle_settings(cam, DEG), sc["means3D"],
                                                                sc["opacities"], shs=sc["shs"], scales=sc["scales"],
                                                                rotations=sc["rotations"])["cov2d"])
    cond = a * c / (a * c - b * b)
    assert (cond > 200).all(), cond                   # the rows really are near-singular (ball scenes: < 10)
    for seed in (5, 6):                               # the error depends on the structure of the incoming gradient
        _, cu, want, _ = full_frame(sc, cam, "room_small", seed=seed)
        sing = np.arange(P0, P0 + len(rows))
        for k in GRADS:
            e = U.rel_err(cu["grads"][k][sing], want[k][sing])
            print("near_singular rows", seed, k, e)
            assert e < B.BWD_REL, (k, e)


def _disparity_fp64(da, focal):
    """scene_gaussian.py:871-881 in fp64."""
    depth, alpha = da[0].double(), da[1].double()
    disp = focal / (depth + alpha * 10 + 1e-5)
    m = alpha <= 0.1
    min_d = disp[m].min() if bool(m.any()) else disp.min()
    return torch.clamp((disp - min_d) / (disp.max() - min_d), 0.0, 1.0)


@pytest.mark.parametrize("route", ["assemble_views", "render_scene"])
def test_production_routes_match_the_oracle(route):
    """assemble_scene + rasterize_views and render_scene (activations inside project_sh), augmentation off, 4 views of
    the small room, one of them the wall camera: each view's image and radii against the oracle, every raw leaf's
    gradient (summed over the views) against the fp64 oracle chained through the reference's activations."""
    from dreamscene_b200.multiview import rasterize_views
    from dreamscene_b200.postprocess import disparity_from_depth_alpha
    from dreamscene_b200.scene import assemble_scene, render_scene
    size = 192
    cams = views(size)
    dev = torch.device("cuda", torch.cuda.current_device())
    groups = room.build_scene(dev, M=M, **SMALL)
    named = room.named_groups(groups)
    S = [U.cuda_settings(c, DEG, device=dev) for c in cams]
    P = sum(int(g["xyz"].shape[0]) for g in groups)
    screens = [torch.zeros(P, 3, device=dev, requires_grad=True) for _ in cams]
    with torch.no_grad():      # the activated inputs both routes rasterize; the oracle reads these
        xyz, op, scl, rot, shs = assemble_scene(named, shs_aug=False, scale_aug=False, noise="fused")
    sc = {"means3D": xyz.cpu(), "opacities": op.cpu(), "shs": shs.cpu(), "scales": scl.cpu(), "rotations": rot.cpu()}
    if route == "render_scene":
        outs, scales_v = render_scene(named, S, shs_aug=False, scale_aug=False, means2D=screens, return_scales=True)
        for v in range(len(cams)):     # render_scene activates inside project_sh: the same scales bit for bit
            assert torch.equal(scales_v[v].detach(), scl)
    else:
        m, o, s_, r, sh = assemble_scene(named, shs_aug=False, scale_aug=False, noise="fused")
        outs = rasterize_views(S, m, o, shs=[sh] * len(cams), scales=[s_] * len(cams), rotations=r, means2D=screens)
    w = [incoming(size, size, 40 + v) for v in range(len(cams))]
    loss = sum((w[v][0].to(dev) * o[0]).sum() + (w[v][1].to(dev) * o[2]).sum() for v, o in enumerate(outs))
    loss.backward()
    torch.cuda.synchronize()
    g_act = {k: torch.zeros_like(v, dtype=torch.float64) for k, v in sc.items()}
    for v, (cam, o) in enumerate(zip(cams, outs)):
        ref32 = run_oracle(sc, cam, DEG, record=True)
        np.testing.assert_array_equal(o[1].cpu().numpy(), ref32["radii"].numpy())
        stats = PT.forward_stats(o[0], o[2], ref32["color"], ref32["depth_alpha"])
        B.check_forward("room_small", stats)
        tiles = [t for t in range(len(ref32["ranges"])) if ref32["ranges"][t, 1] > ref32["ranges"][t, 0]]
        want = PT.oracle_backward_on_tiles(sc, cam, DEG, tiles, w[v][0], w[v][1], ref32["decisions"],
                                           blend=ref32["decisions"]["blend"])
        e = U.rel_err(screens[v].grad.cpu(), want["means2D"])
        assert e < B.BWD_REL, ("means2D", v, e)
        for k in g_act:
            g_act[k] += want[k].reshape(g_act[k].shape)
        # the fused disparity on an almost entirely opaque render, against the reference expression in fp64
        focal = 1 / (2 * math.tan(cam.FoVx / 2))
        disp, _ = disparity_from_depth_alpha(o[2].detach(), focal)
        assert float((o[2][1] <= 0.1).float().mean()) > 0.9
        d64 = _disparity_fp64(o[2].detach().cpu(), focal)
        assert float((disp.cpu().double().reshape(d64.shape) - d64).abs().max()) < 1e-5
    # chain the oracle's activated-input gradients through the reference activations in fp64
    leaves = [{k: v.detach().cpu().double().requires_grad_(True) for k, v in g.items()} for g in named]
    from harness.scene_ref import reference_assemble
    acts = reference_assemble(leaves)
    torch.autograd.backward(list(acts), [g_act["means3D"], g_act["opacities"], g_act["scales"], g_act["rotations"],
                                         g_act["shs"]])
    errs = {}
    for name in named[0]:
        got = torch.cat([g[name].grad.detach().cpu().reshape(-1) for g in named])
        ref = torch.cat([lf[name].grad.reshape(-1) for lf in leaves])
        errs[name] = U.rel_err(got, ref)
    print(route, errs)
    for name, e in errs.items():
        assert e < B.BWD_REL, (name, e)


def test_cfg5_at_full_size_matches_the_oracle_on_sampled_tiles():
    """cfg5 itself (2.63 M Gaussians, 512 x 512), two cameras: complete sorted lists bit-exact, the forward on 24
    list-length-stratified tiles, the COMPLETE gradients with the incoming gradients masked to those tiles."""
    from tests.test_gpu_fullsize import _arbitrate_radii
    from dreamscene_b200 import rasterizer as R
    sc = room.rasterizer_inputs(room.build_scene("cpu", M=M))
    P, size = sc["means3D"].shape[0], 512
    dev = torch.device("cuda", torch.cuda.current_device())
    t = {k: v.to(dev) for k, v in sc.items()}
    for k, cam in enumerate([room.scene_camera(0, size, "cpu"), room.scene_camera(5, size, "cpu")]):
        S = U.cuda_settings(cam, DEG, device=dev)
        with torch.no_grad():
            color, radii, da, _, st = R._forward_impl(S, t["means3D"], t["shs"], None, t["opacities"], t["scales"],
                                                      t["rotations"], None)
        torch.cuda.synchronize()
        S_o, pre, keys, pl, ranges, odec = PT.oracle_lists(sc, cam, DEG)
        _arbitrate_radii(sc, cam, radii.cpu().numpy(), pre["radii"].numpy())
        dec = U.decode_saved(st.saved, P, size, size, st.capacity)
        assert dec["num_pairs"] == len(pl)
        np.testing.assert_array_equal(dec["idx"], pl)
        np.testing.assert_array_equal(dec["tile_start"][:-1], ranges[:, 0])
        np.testing.assert_array_equal(dec["depth_bits"], (keys & np.uint64(0xFFFFFFFF)).astype(np.uint32))
        tiles = PT.sample_tiles(ranges, 24)
        mask = PT.tile_mask(tiles, size, size)
        with torch.no_grad():
            oc, oda, onc, _ = O.composite(pre, pl, ranges, S_o, tiles=tiles)
        stats = PT.forward_stats(color, da, oc, oda, cu_nc=dec["n_contrib"], ref_nc=onc.numpy(), mask=mask)
        B.check_forward("room_cfg5", stats)
        g = torch.Generator().manual_seed(21 + k)
        gc = torch.randn(3, size, size, generator=g) / (size * size) * mask
        gd = torch.randn(2, size, size, generator=g) / (size * size) * mask
        blend = PT.record_blend_decisions(pre, odec, S_o, tiles)
        want = PT.oracle_backward_on_tiles(sc, cam, DEG, tiles, gc, gd, odec, group=3, blend=blend)
        got = PT.cuda_forward_backward(sc, cam, DEG, gc, gd, device=dev)
        errs = PT.grad_errors(got["grads"], want)
        print("cfg5", k, {c: stats[c]["max_abs"] for c in ("color", "depth", "T")},
              stats["n_contrib"]["n_mismatch"], {n: errs[n]["rel_l2"] for n in GRADS})
        for n in GRADS:
            assert errs[n]["rel_l2"] < B.BWD_REL, (n, errs[n])
