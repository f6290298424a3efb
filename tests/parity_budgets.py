"""Forward outlier budgets for the CUDA-vs-oracle comparison, per BASELINE configuration.

north_star: forward RGB/depth/alpha within 1e-4 abs.  alpha >= 1/255 and T < 1e-4 are
discontinuous tests, so two fp32 implementations whose exp() differ in the last bits CAN disagree
on a (pixel, Gaussian) pair; such a pixel is then off by up to one blend weight.  The budgets are
tied to what tools/parity_stats.py measured on an H100 (variant "default" = ex2.approx/rcp.approx): at all
four configurations - 196 608 values (cfg1, whole frame), 786 432 (cfg2 and cfg2b, whole frame), 73 728 (cfg3,
96 sampled tiles) - the measured number of values off by more than 1e-4 is ZERO, the largest |diff| is 6.6e-7
(colour), 2.9e-6 (depth, which is an un-normalised view-depth sum) and 3.0e-7 (T), and n_contrib has zero mismatches.  With nothing
measured to multiply by three, the budgets allow one discontinuity event per 1e5 values (so a
borderline pair flipping on another seed or GPU does not fail the suite), each bounded by one blend
weight, and are otherwise 30x above the measured maxima.

    frac  = fraction of compared values with |cuda - oracle| > 1e-4
    maxab = largest |cuda - oracle|
"""
FWD_ATOL = 1e-4
BWD_REL = 1e-3          # north_star: backward gradients within 1e-3 relative (norm-wise); measured <= 1.1e-5
                        # when the fp64 oracle replays the fp32 blend decisions (4.3e-4 at cfg1 otherwise:
                        # ONE borderline pair decided differently by fp64, see DESIGN.md section 1)

_B = {"color": (1e-5, 6e-3), "depth": (1e-5, 3e-2), "T": (1e-5, 6e-3), "n_contrib": 1e-5}
# config -> channel -> (max frac_bad, max abs)
BUDGETS = {name: dict(_B) for name in ("cfg1_10k_256", "cfg2_100k_512", "cfg2b_81920_512", "cfg3_1M_1024",
                                         "room_cfg5")}
# room_small (tests/test_gpu_room.py: 49 800 Gaussians seen from inside the room, whole frames of 200^2 and 256^2, plus
# the constructed edge Gaussians): opaque views with lists of up to 3 000 entries per tile hold more borderline
# (pixel, Gaussian) pairs than the ball scenes.  Measured on an H100: up to 2 of 110 592 colour values (1.8e-5) and 1
# of 36 864 depth values off by more than 1e-4, each a single alpha >= 1/255 decision (largest |diff| 3.8e-4, below
# one blend weight); otherwise colour <= 9.0e-5, depth <= 1.4e-4, T <= 6.7e-5, no n_contrib mismatch, gradients within
# 1.5e-4 over the frame and 5.7e-4 over the near-singular rows alone (frames of 192^2, 200^2 and 256^2).  The budget
# allows four such events per 36 864-pixel frame (1e-4), each bounded by one blend weight as above.
BUDGETS["room_small"] = {"color": (1e-4, 6e-3), "depth": (1e-4, 3e-2), "T": (1e-4, 6e-3), "n_contrib": 1e-4}
# room_cfg5 (2.63 M Gaussians, 512^2, 24 sampled tiles per view) shares the ball budgets: measured on an H100, zero values
# off by more than 1e-4, largest |diff| 7.7e-7 (colour), 2.1e-6 (depth), 2.4e-7 (T), no n_contrib mismatch, gradients
# within 1.5e-5.


def check_forward(config, stats):
    b = BUDGETS[config]
    for chan in ("color", "depth", "T"):
        frac, mx = b[chan]
        s = stats[chan]
        assert s["frac_bad"] <= frac, f"{config}/{chan}: {s['n_bad']} of {s['n']} values off by > {FWD_ATOL} (budget {frac})"
        assert s["max_abs"] <= mx, f"{config}/{chan}: max abs diff {s['max_abs']} (budget {mx})"
    if "n_contrib" in b and "n_contrib" in stats:
        s = stats["n_contrib"]
        assert s["frac_mismatch"] <= b["n_contrib"], f"{config}/n_contrib: mismatch rate {s['frac_mismatch']}"
