"""TEST INFRASTRUCTURE ONLY -- comparison of gradients with a float64 oracle that ran with the LeakyReLU masks of the computation under
test (oracle/shade_oracle.py, `slopes=`).  Once the masks agree, nothing but rounding separates the two, so every point and every MLP
tensor is held to one strict bound relative to its tensor's scale, without an allowance for outliers.

The one exception is points_conf of point 0: every empty neighbour slot gathers point 0 (clamp(pidx, 0), neural_points.py:707), so
a loss on conf_coefficient adds one term per padded slot into it, tens of thousands in an fp32 sum.  Its bound follows from that count.
"""
import ctypes as C

import numpy as np
import torch

from . import forward_check

LAYERS = ("block1.0", "block1.2", "block3.0", "block3.2", "color_branch.0", "color_branch.2", "color_branch.4")
U32 = 2.0 ** -24    # unit roundoff of fp32

# (points, MLP tensors): the largest error allowed, relative to the tensor's scale, per (pnb_bwd_fp32 mode, pnb_precision), 4-5x the
# largest measured over tests/test_gpu_grad_f64.py's cases on an H100 80GB HBM3 at a 400 W power limit:
#   mode 0 (BF16x3 recompute, dX, dW)    bf16x3: points 8.9e-6, MLP 2.8e-5    fp32: points 8.3e-6, MLP 2.7e-5
#   mode 4 (fp32 recompute, BF16x3 dX/dW) bf16x3: points 8.8e-6, MLP 2.6e-5
#   mode 1 (fp32 CUDA-core GEMMs)         bf16x3: points 4.7e-6, MLP 1.2e-6    fp32: points 4.9e-7, MLP 6.7e-7
# The cases below the rotated-camera ones (background, raydist_mode_unit 0, saturated rays, random conf_coefficient weights, frozen groups,
# checkpoint value ranges; H100 80GB HBM3 at 700 W) measured at most: tensor-core modes points 1.3e-5, MLP 2.8e-5; mode 1 points 5.5e-6,
# MLP 3.5e-6 (both in raydist_mode_unit 0 at SR 80).
# The tensor-core dX / dW GEMMs carry the ~1e-5 of the BF16x3 split (tests/test_gpu_umma.py); in mode 1 the points see the BF16x3
# forward's (sigma, rgb), from which the composite backward starts.  One flipped or lost pair row moves its points by ~1e-3 of scale.
# The exact-count cases (batches of 1 to 2049 valid samples or 1 to 4097 pair rows, S_TARGETS / P_TARGETS; H100 80GB HBM3 at 700 W)
# measured at most: mode 0 points 3.0e-5, MLP 2.0e-5 (fp32 forward 1.0e-5, 1.7e-5); mode 4 points 3.3e-5, MLP 2.1e-5; mode 1 points
# 1.9e-6, MLP 3.2e-6 (fp32 forward 6.0e-7, 2.7e-6).  The largest tensor-core errors are one-ray batches whose every valid sample has
# a single neighbour (S = P = 8 and 9): each point's gradient comes from one pair row, so nothing averages the BF16x3 error of its
# chain of GEMMs down.
RTOL = {(0, "bf16x3"): (4e-5, 1.2e-4), (0, "fp32"): (4e-5, 1.2e-4), (4, "bf16x3"): (4e-5, 1.2e-4),
        (1, "bf16x3"): (2e-5, 5e-6), (1, "fp32"): (2e-6, 3e-6)}

# The frustum query's opaque surface (scene.FRUSTUM_CONFIGS["dtu_surface"], alpha bias +300: sigma ~300) in the colour-only checks
# (tests/test_gpu_frustum_fused.py, the F 63 leg of tests/test_gpu_feedforward.py) and in tests/test_gpu_frustum_f64.py: the MLP
# tensors per (mode, precision).  RTOL, except mode 1 with the BF16x3 forward: 4.6x the 5.4e-6 measured there (block3.2.weight; the
# composite backward starts from the BF16x3 (sigma, rgb), whose per-sample error grows with sigma), above RTOL's mode-1 bound of the
# tiny world scene.  H100 80GB HBM3 at a 700 W power limit.
FRUSTUM_MLP_RTOL = {(0, "bf16x3"): RTOL[(0, "bf16x3")][1], (4, "bf16x3"): RTOL[(4, "bf16x3")][1], (1, "bf16x3"): 2.5e-5,
                    (0, "fp32"): RTOL[(0, "fp32")][1], (1, "fp32"): RTOL[(1, "fp32")][1]}
# alpha_branch.0 with agg_intrp_order 1: a sum over the valid samples of dL/dz [1, h-bar] (z: sigma's pre-activation).  On the opaque
# surface with a colour loss its terms cancel (sum |terms| 9-17x the largest entry in tests/test_gpu_frustum_fused.py), so its error
# scales with sum |terms|, not with the result: each term carries the relative error of the (sigma, rgb) it starts from.  Measured
# relative to each entry's sum |terms| (sum_error), the largest over the three files:
#   BF16x3 forward, modes 0 / 4 / 1   2.0e-5 (alpha_branch.0.weight; the same in every mode)
#   fp32 forward, mode 0              7.6e-6
#   fp32 forward, mode 1              2.9e-6 (every GEMM and the forward in fp32)
# The fp32 forward takes the mode-1 error from 1.6e-5 to 2.9e-6 of sum |terms|: most of it is the BF16x3 forward's.  Bounds 4-5x.
ALPHA1_SUM_RTOL = {(0, "bf16x3"): 9e-5, (4, "bf16x3"): 9e-5, (1, "bf16x3"): 9e-5, (0, "fp32"): 3.5e-5, (1, "fp32"): 1.3e-5}
# ... and relative to the tensor's scale, so that no entry is held looser than by a plain bound: measured 1.2e-4 (BF16x3 forward,
# tests/test_gpu_feedforward.py, every mode) and 1.7e-5 (fp32 forward); 3e-4 is the bound these tests had in modes 4 and 1, 8e-5 is
# 4.6x the fp32 forward's.
ALPHA1_RTOL = {"bf16x3": 3e-4, "fp32": 8e-5}


def rel_point_errors(a, ref):
    """[N] largest |a - ref| of each point (over its channels) relative to max |ref| of the tensor.  a, ref: [1,N,C] or [N,C]."""
    a = np.asarray(a, np.float64)
    ref = np.asarray(ref, np.float64).reshape(a.shape)
    a, ref = a.reshape(-1, a.shape[-1]), ref.reshape(-1, a.shape[-1])
    scale = max(np.abs(ref).max(), 1e-30)
    return np.abs(a - ref).max(axis=-1) / scale


def rel_error(a, ref):
    a = np.asarray(a, np.float64)
    ref = np.asarray(ref, np.float64).reshape(a.shape)
    return float(np.abs(a - ref).max() / max(np.abs(ref).max(), 1e-30))


def check_points(a, ref, name, rtol):
    """Every point within rtol of the tensor's scale.  Returns the largest relative error."""
    e = rel_point_errors(a, ref)
    bad = np.nonzero(e > rtol)[0]
    assert bad.size == 0, "%s: %d points beyond %.1e of scale (worst %.3e at point %d)" % (name, bad.size, rtol, e.max(), int(e.argmax()))
    return float(e.max())


def sum_error(a, ref, abs_terms):
    """Largest |a - ref| of a gradient tensor that is a sum over samples, relative to the larger of the tensor's scale (max |ref|) and
    the entry's sum of absolute terms (abs_terms, broadcast to a's shape).  Where the terms cancel, each term's own error (the
    forward's ~1e-5 of the BF16x3 split, which the backward starts from) adds up over sum |terms|, not over the result."""
    a = np.asarray(a, np.float64)
    ref = np.asarray(ref, np.float64).reshape(a.shape)
    scale = np.maximum(np.broadcast_to(np.asarray(abs_terms, np.float64), a.shape), max(np.abs(ref).max(), 1e-30))
    return float((np.abs(a - ref) / scale).max())


def point0_conf_bound(n0, ref0, term=1e-3):
    """Bound of the error of an fp32 sum into point 0's conf gradient: n0 terms (one per gathered slot), each rounding step off by at
    most U32 of the partial sum, which stays below |ref0| plus the padded terms' `term` each (1e-3: the loss's
    1e-3 * conf_coefficient.sum())."""
    return n0 * U32 * (abs(float(ref0)) + term * n0)


def check_conf(a, ref, n0, rtol):
    """points_conf: points 1.. within rtol of their scale (point 0 left out of it: its padded terms would dominate the scale), point 0
    within point0_conf_bound.  n0: number of [R',SR,K] slots whose clamped index is 0.  Returns the largest relative error of 1.."""
    a = np.asarray(a, np.float64).reshape(-1)
    ref = np.asarray(ref, np.float64).reshape(-1)
    e = check_points(a[1:, None], ref[1:, None], "points_conf (points 1..)", rtol)
    d0, b0 = abs(a[0] - ref[0]), point0_conf_bound(n0, ref[0])
    assert d0 <= b0, "points_conf of point 0: |diff| %.3e > %.3e (%d accumulated terms)" % (d0, b0, n0)
    return e


class MaskRecorder:
    """Stands in for torch.nn.functional in oracle/shade_oracle.py (monkeypatch its `F`): records the slope each LeakyReLU unit takes
    (1 above zero, else the negative slope, as torch's derivative does) in call order, which is the layer order of `slopes=`."""

    def __init__(self, functional):
        self._f, self.slopes = functional, []

    def __getattr__(self, k):
        return getattr(self._f, k)

    def leaky_relu(self, x, negative_slope):
        self.slopes.append(torch.where(x > 0, 1.0, negative_slope).to(torch.float64).detach())
        return self._f.leaky_relu(x, negative_slope)


def flipped_rows(slopes_a, slopes_b):
    """Per layer, the rows in which some unit has a different slope in the two mask sets."""
    return [(sa != sb).any(dim=-1) for sa, sb in zip(slopes_a, slopes_b)]


# Batch sizes at which the backward's launch geometry changes (backward.cu, gemm_tc.cu), as exact counts of valid samples S (n_valid)
# and of pair rows P (n_pairs):
#   S: one warp per valid sample, 8 per block (k_bwd_build, k_bwd_reduce_fwd / _bwd): 1, 8, 9; 128-row output tiles of the colour GEMMs
#      (M = S): 127, 128, 129; 256-row slabs of k_bwd_head, k_dw_small<3>, k_bwd_alpha_params_o1: 255, 256, 257; 512-row slabs of
#      k_colsum4: 511, 512, 513; blocks of 1024 of exclusive_scan_u32 over the per-sample pair counts: 1024, 1025; the colour dW
#      split-K (max(2, ceil(S / 2048)) splits) and 2048-row slabs of k_colsum / k_gemm<true>: 2048, 2049
#   P: the dW split-K's single-split fallback (kchunk rounded up to 32): 1, 32, 33; 128-row tiles of the pair GEMMs (M = P): 127, 128,
#      129; 256-row slabs of k_bwd_alpha_params: 255, 256, 257; split-K and 2048-row slabs: 2047, 2048, 2049, 4096, 4097
S_TARGETS = (1, 8, 9, 127, 128, 129, 255, 256, 257, 511, 512, 513, 1024, 1025, 2048, 2049)
P_TARGETS = (1, 32, 33, 127, 128, 129, 255, 256, 257, 2047, 2048, 2049, 4096, 4097)
SPLITK_ROWS, SPLITK_MAX = 2048, 64


def dw_splits(rows):
    """(splits gemm_tn_acc asks for, splits gemm_tc runs) of a dW GEMM over `rows` reduction rows: max(2, ceil(rows / 2048)) capped at
    64, then kchunk = that share rounded up to 32 rows and the count recomputed (1 for 1..32 rows: one split through the workspace)."""
    asked = min(max(2, -(-rows // SPLITK_ROWS)), SPLITK_MAX)
    kchunk = -(-(-(-rows // asked)) // 32) * 32
    return asked, -(-rows // kchunk)


def ray_census(sample_pidx, ray_mask):
    """Per hit ray of a query (sample_pidx [R',SR,K] of the hit rays, ray_mask [R]): its index among the R rays, its valid samples (slots
    with a neighbour: the rows of n_valid) and its pairs (filled K slots: the rows of n_pairs)."""
    v = np.asarray(sample_pidx) >= 0
    return dict(rays=np.nonzero(np.asarray(ray_mask))[0], S=v.any(-1).sum(-1), P=v.sum((-2, -1)))


def select_rays(counts, target):
    """Positions (ascending) of entries of counts [n] (non-negative integers) that sum to `target` exactly, or None if no subset does.
    Subset-sum over the prefix of the entries it needs: among the subsets, the one that skips every entry it can from the back, so
    that a target reached by a prefix of the rays takes that prefix."""
    c = np.asarray(counts, np.int64)
    if target < 0 or target > int(c.sum()):
        return None
    n = int(np.searchsorted(np.cumsum(c), target)) + 1 if target > 0 else 0
    while True:
        n = min(n, len(c))
        reach = np.zeros((n + 1, target + 1), bool)        # reach[i][s]: some subset of the first i entries sums to s
        reach[0, 0] = True
        for i in range(n):
            reach[i + 1] = reach[i]
            if c[i] <= target:
                reach[i + 1, c[i]:] |= reach[i, :target + 1 - c[i]]
        if reach[n, target] or n == len(c):
            break
        n *= 2
    if not reach[n, target]:
        return None
    pick, s = [], target
    for i in range(n, 0, -1):
        if not reach[i - 1, s]:
            pick.append(i - 1)
            s -= int(c[i - 1])
    return np.array(pick[::-1], np.int64)


_CENSUS = {}


def frame_census(cfg_name, rotated=False, device="cuda:0", **over):
    """ray_census of the whole frame of scene.CONFIGS[cfg_name] (camera scene.orbit_rotation() if rotated, query options `over` of
    harness.make_opt), from the drop-in's own query export, plus the pixel of every hit ray.  Cached per arguments."""
    key = (cfg_name, rotated, device, tuple(sorted(over.items())))
    if key not in _CENSUS:
        from pointnerf_b200 import harness, scene
        from pointnerf_b200.point_query import make_cam_opts
        cfg = scene.CONFIGS[cfg_name]
        net, _, _ = harness.build_model(cfg, device, **over)
        rays = scene.make_rays(cfg, None, camrotc2w=scene.orbit_rotation() if rotated else None)
        r = {k: v.to(device) for k, v in rays.items()}
        with torch.no_grad():
            net(r["campos"], r["raydir"], bg_color=r["bg_color"], camrotc2w=r["camrotc2w"], pixel_idx=r["pixel_idx"], near=r["near"],
                far=r["far"], h=r["h"], w=r["w"], intrinsic=r["intrinsic"])
        net.check_errors()
        q = net.last
        ex = q.export(make_cam_opts(list(q.desc.campos), rays["camrotc2w"][0]), want_pers=False, want_dirs=False)
        c = ray_census(ex["sample_pidx"].cpu().numpy(), ex["ray_mask"].cpu().numpy())
        assert int(c["S"].sum()) == int(q.counters["n_valid"]) and int(c["P"].sum()) == int(q.counters["n_pairs"])
        c["pixels"] = rays["pixel_idx"][0].numpy()[c["rays"]]
        _CENSUS[key] = c
    return _CENSUS[key]


def pixels_for(census, count, target):
    """The pixels of a subset of the census's hit rays whose valid samples (count "S") or pairs (count "P") add up to target exactly."""
    pick = select_rays(census[count], target)
    assert pick is not None, "no subset of the frame's hit rays has %s = %d (the frame holds %d)" % (count, target, int(census[count].sum()))
    return census["pixels"][pick]


def kernel_masks(net, q, F, camrotc2w):
    """After a forward and backward of `net` (query `q`, point_features_dim F): the backward's masks as `slopes=` of the oracle (pair
    rows in the flattened [R',SR,K] order of sample_pidx >= 0, colour rows per sample slot), the dense export of the query, and the
    pair-row count."""
    from pointnerf_b200 import lib
    from pointnerf_b200.point_query import make_cam_opts
    l = lib.load()
    S, P = int(q.counters["n_valid"]), int(q.counters["n_pairs"])
    out = (C.c_void_p * 10)()
    ws = net._bwd_ws
    lib.check(l.pnb_backward_tables(ws.data_ptr(), ws.numel(), S, q.desc.cap_samples, F, out), "pnb_backward_tables")
    dev_view = forward_check.dev_view
    H = [dev_view(ws, out[0], torch.float32, (P, 256)), dev_view(ws, out[1], torch.float32, (P, 272))[:, :256],
         dev_view(ws, out[2], torch.float32, (P, 256)), dev_view(ws, out[3], torch.float32, (P, 256))]
    Cc = [dev_view(ws, out[i], torch.float32, (S, 128)) for i in (4, 5, 6)]
    pair_off = dev_view(ws, out[7], torch.int32, (S + 1,)).long()
    row_samp = dev_view(ws, out[8], torch.int32, (P,)).long()
    pidx = dev_view(ws, out[9], torch.int32, (P,)).long()
    ex = q.export(make_cam_opts(list(q.desc.campos), camrotc2w), want_pers=False, want_dirs=False)
    SR = q.SR
    # valid sample -> (ray, sample slot) -> its row of the export; pair row -> (its sample, K slot)
    srow = forward_check.sample_map(q, ex)["srow"]
    flat = forward_check.pair_map(dict(srow=srow), pair_off, row_samp, pidx, ex, q.K)
    order = torch.argsort(flat)
    slopes = [torch.where(h[order] > 0, 1.0, 0.01).double() for h in H]
    for c in Cc:
        s = torch.ones(ex["sample_pidx"].shape[0] * SR, 128, dtype=torch.float64)
        s[srow] = torch.where(c > 0, 1.0, 0.01).double()
        slopes.append(s)
    return slopes, ex, P
