"""GPU: the workloads bench.py times, at the sizes it times them, against float64.

The other float64 files hold every kernel to float64 on small clouds and contiguous centre patches.  This file checks what the bench
lines measure, at their own sizes, with the same method and bounds:

A. The training step (bench.py train_section: `train` on ship_optimise, N = 600k, and `scannet` on scannet_8gpu, N = 5M, P = 30, the
   camera inside a box, near 0.1).  The bench's first batch: 3600 pixels from RandomState(0) over the whole view, train jitter on,
   parallel.TrainStep(world=1).gradients() (forward + backward, no Adam).  The float64 reference is autograd through
   oracle/shade_oracle_rw2c.py on the kernel's own query export (the jittered sample positions) with the backward's own LeakyReLU
   masks (grad_check.kernel_masks), on TrainStep's loss: the squared colour errors over the global count, plus 1e-4 x the zero-one
   term over its count, the counts held constant.  The oracle runs on the host one chunk of rays at a time (the loss is a sum over
   rays), on the rows of the points the batch gathers only.  Every gathered point row is held to grad_check.RTOL of its tensor's
   scale, every other row of the 600k or 5M must be exactly zero, bit for bit, the 18 MLP tensors to RTOL, points_conf of point 0 to
   grad_check.point0_conf_bound, and the loss to float64; no outlier allowance.  Scattered rays spread every point's atomic adds over
   many tiles, and scannet's touched points lie above 2^22.  Neither bench step reaches the split-K cap of the dW GEMMs (64 slabs of
   2048 pair rows), so scannet's first two batches also run as one step, which does.  Ship also runs with F = 63 (bench_feat63.py's
   training leg: point_features_dim 63, point modes 01) in modes 0, 4 and 1 on the same batch.
B. The forward, sample by sample (tests/test_gpu_forward_f64.py's `_run` and its table), on seeded sets of 1024 pixels over the whole
   truck_8gpu, scannet_8gpu and lego_render frames, with the frozen, general and fp32 kernels; truck adds the image-corner strip of
   tests/test_gpu_shade.py.  lego_render also runs with F = 63 (bench_feat63.py's render leg) and with scene.edit_frames' per-point
   frames (bench_rw2c.py).  Every row of the frozen cloud's `pre` table is compared with float64, in row chunks.
C. The whole frame (runner.render_image, as the bench renders it) equals render_full on B's pixel subset bit for bit, which equals
   forward()'s result on its hit rays: B's float64 check covers the frame the bench renders.

Measured on an H100 80GB HBM3 at a 700 W power limit: see DESIGN §6 ("The benchmarked workloads at their sizes").
"""
import contextlib
import gc
import math
import time
import traceback

import numpy as np
import pytest
import torch

import test_gpu_forward_f64 as fwd
from oracle import grad_check, shade_oracle, shade_oracle_rw2c
from pointnerf_b200 import harness, parallel, runner, scene

pytestmark = pytest.mark.gpu
DEV = "cuda:0"
BATCH = 3600                 # rays per step (bench.py train_section)
ZERO_ONE_WEIGHT = 1e-4       # parallel.TrainStep's weight of the zero-one term
POINT_KEYS = ("embedding", "color", "dir", "conf")
CHUNK_RAYS = 256             # rays per float64 oracle chunk (~40k pairs on scannet)


# ---- the method (also run on the CPU by tests/test_bench_scale_method.py) ----
def touched_rows(pidx):
    """Sorted ids of the points a batch gathers: every valid neighbour, and point 0, which every empty slot gathers."""
    return torch.unique(torch.cat([torch.zeros(1, dtype=torch.long), pidx[pidx >= 0].long()]))


def pair_offsets(pidx):
    """[R'+1] first row of each ray among the pair rows of `slopes=` (the flattened [R',SR,K] order of sample_pidx >= 0)."""
    n = (pidx >= 0).reshape(pidx.shape[0], -1).sum(-1)
    return torch.cat([torch.zeros(1, dtype=torch.long), torch.cumsum(n, 0)])


def ray_chunks(n_rays, size):
    return [(r0, min(r0 + size, n_rays)) for r0 in range(0, n_rays, size)]


def _slopes(s):
    """A layer's slopes from a boolean mask (True: slope 1) as grad_check.kernel_masks builds them, or a float one unchanged."""
    return torch.where(s, 1.0, shade_oracle.LEAKY_SLOPE).double() if s.dtype == torch.bool else s


def train_loss(ray_color, gt, conf_coefficient, n_se, n_zo):
    """parallel.TrainStep's loss on one set of rays, with the global counts n_se (colour terms) and n_zo (conf_coefficient entries)."""
    se = ((ray_color - gt) ** 2).sum()
    zo = (-torch.log(conf_coefficient + 1e-3)).sum()
    return se / n_se + ZERO_ONE_WEIGHT * zo / n_zo


def reference_gradients(points, mlp, pidx, loc_w, raydir_hit, gt_hit, campos, cam, vsize, bg, slopes, n_se, n_zo, chunks,
                        agg_intrp_order=2, raydist_mode_unit=1):
    """float64 autograd of train_loss through oracle/shade_oracle_rw2c.py with the given masks, one chunk of rays at a time.

    points: xyz [N,3], embedding / color / dir / conf [1,N,C], Rw2c; only the rows touched_rows(pidx) enter, so that a chunk's backward
    costs its own pairs and not N.  slopes: the 7 layers of shade()'s `slopes=` for the whole batch (float, or bool with True = 1);
    each chunk takes the pair rows and sample rows of its own rays.  chunks: (r0, r1) ranges of the R' rays, whose gradients are added.
    Returns (gradients: the four point tensors [1,U,C] on the touched rows and the 18 MLP tensors, keep [U], loss)."""
    keep = touched_rows(pidx)
    cpidx = torch.where(pidx >= 0, torch.searchsorted(keep, pidx.long().clamp(min=0)), -1)
    leaves = {k: points[k][:, keep].double().requires_grad_(True) for k in POINT_KEYS}
    R = points["Rw2c"]
    pts = dict(xyz=points["xyz"][keep].double(), Rw2c=(R[keep] if R.dim() == 3 else R).double(), **leaves)
    w = {k: v.double().requires_grad_(True) for k, v in mlp.items()}
    poff, SR = pair_offsets(pidx), pidx.shape[1]
    loss = 0.0
    for r0, r1 in chunks:
        p0, p1 = int(poff[r0]), int(poff[r1])
        sl = [_slopes(s[p0:p1]) for s in slopes[:4]] + [_slopes(s[r0 * SR:r1 * SR]) for s in slopes[4:]]
        sh = shade_oracle_rw2c.shade(pts, w, cpidx[r0:r1], loc_w[r0:r1], raydir_hit[r0:r1], campos, cam, vsize, bg, dtype=torch.float64,
                                     agg_intrp_order=agg_intrp_order, slopes=sl, raydist_mode_unit=raydist_mode_unit)
        lc = train_loss(sh["ray_color"], gt_hit[r0:r1].double(), sh["conf_coefficient"], n_se, n_zo)
        lc.backward()
        loss += float(lc.detach())
    grads = {k: v.grad for k, v in leaves.items()}
    grads.update({k: v.grad for k, v in w.items()})
    return grads, keep, loss


def point0_term(conf, n_zo):
    """Gradient of one empty slot's zero-one term into points_conf of point 0 (the slot gathers point 0's clamped conf)."""
    c0 = min(max(float(conf.reshape(-1)[0]), 1e-4), 1.0)
    return ZERO_ONE_WEIGHT / (n_zo * (c0 + 1e-3))


def step_errors(got, ref, keep, n0, term):
    """got: the computation's gradients (the four point tensors [1,N,C] on any device, the MLP tensors); ref, keep: reference_gradients.
    Returns {name: largest error relative to the tensor's scale} over the touched rows and the MLP tensors, the points_conf of point 0
    as (|error|, its bound), and per point tensor the number of untouched rows with a non-zero bit."""
    err, untouched = {}, {}
    for k in POINT_KEYS:
        g = got[k].reshape(-1, got[k].shape[-1])
        mask = torch.ones(g.shape[0], dtype=torch.bool, device=g.device)
        mask[keep.to(g.device)] = False
        untouched[k] = int(((g.view(torch.int32) != 0).any(-1) & mask).sum())
        a, r = g[keep.to(g.device)].cpu().double(), ref[k].reshape(-1, g.shape[-1])
        if k == "conf":          # point 0 (keep[0]) to its own bound: every empty slot adds a term into it
            err[k] = float(grad_check.rel_point_errors(a[1:], r[1:]).max()) if a.shape[0] > 1 else 0.0
            conf0 = (abs(float(a[0, 0] - r[0, 0])), grad_check.point0_conf_bound(n0, r[0, 0], term))
        else:
            err[k] = float(grad_check.rel_point_errors(a, r).max())
    for k in ref:
        if k not in POINT_KEYS:
            err[k] = grad_check.rel_error(got[k].cpu(), ref[k])
    return err, conf0, untouched


def check_step(err, conf0, untouched, rtol):
    """The bounds of step_errors' report: points and MLP tensors within rtol = (points, MLP) of scale, point 0's conf within its bound,
    no untouched row with a non-zero bit."""
    bound = {k: rtol[0 if k in POINT_KEYS else 1] for k in err}
    bad = ["%s: %.3e of scale > %.1e" % (k, v, bound[k]) for k, v in err.items() if not v <= bound[k]]
    if not conf0[0] <= conf0[1]:
        bad.append("points_conf of point 0: %.3e > %.3e" % conf0)
    bad += ["%s: %d untouched rows not zero" % (k, n) for k, n in untouched.items() if n]
    assert not bad, "; ".join(bad)


def loss_bound(loss, mse, delta):
    """|loss - float64| allowed when every ray colour is within delta of float64: sum (e + d)^2 - e^2 over n terms is at most
    n (2 delta rms(e) + delta^2), plus 1e-6 of the loss for the fp32 sums.  A bound of bounds: delta is the forward table's composite
    bound (1e-5), not a measured colour error, so it sits ~3 orders of magnitude above the differences measured (<= 1.4e-8).  It catches a
    wrong count or a missing term of the loss, not a small systematic error of it; the gradients carry the strict comparison."""
    return 2 * delta * math.sqrt(mse) + delta * delta + 1e-6 * abs(loss)


# ---- A. the training step at bench scale ----
@contextlib.contextmanager
def _device_released():
    """A case's 600k / 5M-point model leaves the device whatever the outcome.  Each case's body runs in a function below this one; when
    it fails, pytest keeps the traceback, whose frames would hold the model: their locals are cleared before the error goes on."""
    try:
        yield
    except BaseException as e:
        traceback.clear_frames(e.__traceback__)
        raise
    finally:
        gc.collect()
        torch.cuda.empty_cache()


# Points in mode 1 with the fp32 forward: grad_check.RTOL's 2e-6 is 4x what the tiny cases measured (4.9e-7), where a point's gradient
# sums ~37 pairs.  On ship a point has 1.6 pairs on average and the largest rows are one to three pairs' worth, so the fp32 rounding of
# a single pair's backward shows at the tensor's scale instead of averaging down: measured over jitter draws, 1.3e-6 to 1.7e-6 with
# the fp32 forward and up to 2.4e-6 with the BF16x3 forward (the same backward; points_color, embedding and dir alike, and the same
# with the sample geometry w2pers taken in fp32).  On scannet (5.8 pairs per point) the BF16x3-forward mode-1 case measures 4.2e-7.
# Held to 1e-5, 4x the largest of those; the MLP tensors keep RTOL.
POINTS_RTOL = {(1, "fp32"): 1e-5}


def _rtol(mode, precision):
    pts, mlp = grad_check.RTOL[(mode, precision)]
    return POINTS_RTOL.get((mode, precision), pts), mlp


def _reset_peak_memory():
    torch.cuda.empty_cache()
    torch.empty(1, device=DEV)          # the allocator must exist before its statistics are reset
    torch.cuda.reset_peak_memory_stats(DEV)


def bench_batch(cfg, batches=1):
    """bench.py train_section's first `batches` batches at world 1, as one step: per batch 3600 pixels from RandomState(0) over the
    whole view (x, then y) and the target colours from a Generator seeded 1; raydir and pixel_idx on the device, the camera scalars on
    the host (as the bench hands them over)."""
    rng = np.random.RandomState(0)
    g = torch.Generator().manual_seed(1)
    pix, gt = [], []
    for _ in range(batches):
        px = rng.randint(0, cfg.W, size=(BATCH,)).astype(np.float32)
        py = rng.randint(0, cfg.H, size=(BATCH,)).astype(np.float32)
        gt.append(torch.rand(BATCH, 3, generator=g))
        pix.append(np.stack([px, py], -1))
    rays = scene.make_rays(cfg, np.concatenate(pix))
    kw = {k: (v.to(DEV) if k in ("raydir", "pixel_idx") else v) for k, v in rays.items()}
    return kw, torch.cat(gt), rays


# (config, pnb_bwd_fp32 mode, pnb_precision, bench batches in the step, point_features_dim F).  The bench's scannet step has ~106k pair
# rows (51.6 slabs of 2048), below the split-K cap of the tensor-core dW GEMMs (64 slabs, csrc/backward.cu SPLITK_MAX); its first two
# batches as one step (~211k rows) run the pair layers' dW GEMMs with the cap, every slab taller than 2048 rows.  F = 63 on ship is
# bench_feat63.bench_train's 63-channel leg (the DTU scripts' point_features_dim 63, point modes 01) on the same batches.
TRAIN_CASES = [("ship_optimise", 0, "bf16x3", 1, 32), ("ship_optimise", 4, "bf16x3", 1, 32), ("ship_optimise", 1, "bf16x3", 1, 32),
               ("ship_optimise", 1, "fp32", 1, 32),
               ("scannet_8gpu", 0, "bf16x3", 1, 32), ("scannet_8gpu", 4, "bf16x3", 1, 32), ("scannet_8gpu", 1, "bf16x3", 1, 32),
               ("scannet_8gpu", 0, "bf16x3", 2, 32), ("scannet_8gpu", 4, "bf16x3", 2, 32),
               ("ship_optimise", 0, "bf16x3", 1, 63), ("ship_optimise", 4, "bf16x3", 1, 63), ("ship_optimise", 1, "bf16x3", 1, 63)]


def _train_id(c):
    return "%s-mode%d-%s-x%d" % c[:4] + ("" if c[4] == 32 else "-F%d" % c[4])


@pytest.mark.parametrize("cfg_name,mode,precision,batches,F", TRAIN_CASES, ids=[_train_id(c) for c in TRAIN_CASES])
def test_training_step_gradients(cfg_name, mode, precision, batches, F):
    with _device_released():
        _training_step_case(cfg_name, mode, precision, batches, F)


def _training_step_case(cfg_name, mode, precision, batches, F=32):
    cfg = scene.CONFIGS[cfg_name]
    _reset_peak_memory()
    net, _, opt = harness.build_model(cfg, DEV, alpha_bias=3.0, is_train=True, pnb_precision=precision, pnb_bwd_fp32=mode, feat_dim=F)
    ts = parallel.TrainStep(net, world=1)
    kw, gt, rays = bench_batch(cfg, batches)
    n_rays = batches * BATCH
    torch.manual_seed(0)        # the train jitter (torch.rand on the device): a failure replays; the bounds hold over other draws
    loss = float(ts.gradients(kw, gt.to(DEV)))
    net.check_errors()
    npn = net.neural_points
    N = npn.xyz.shape[0]
    q = net.last
    cam = rays["camrotc2w"][0]
    slopes, ex, P = grad_check.kernel_masks(net, q, F, cam)
    slopes = [s == 1 for s in slopes]         # 1 byte per unit instead of 8; _slopes rebuilds the same values per chunk
    peak = torch.cuda.max_memory_allocated(DEV)
    pidx, loc_w = ex["sample_pidx"].cpu(), ex["sample_loc_w"].cpu()
    hit = ex["ray_mask"].cpu() > 0
    Rn, SR, K = pidx.shape
    n_se, n_zo = 3 * Rn, Rn * SR * K
    assert (float(ts.last["n_hit_terms"]), float(ts.last["n_conf_terms"])) == (n_se, n_zo)
    got = dict(embedding=npn.points_embeding.grad, color=npn.points_color.grad, dir=npn.points_dir.grad, conf=npn.points_conf.grad)
    got.update({k: p.grad for k, p in net.aggregator.named_parameters()})
    points = dict(xyz=npn.xyz.detach().cpu(), Rw2c=torch.eye(3), embedding=npn.points_embeding.detach().cpu(),
                  color=npn.points_color.detach().cpu(), dir=npn.points_dir.detach().cpu(), conf=npn.points_conf.detach().cpu())
    t0 = time.time()
    ref, keep, loss64 = reference_gradients(points, harness.mlp_cpu(net.aggregator), pidx, loc_w, rays["raydir"][0][hit], gt[hit],
                                            rays["campos"][0], cam, opt.vsize, rays["bg_color"][0], slopes, n_se, n_zo,
                                            ray_chunks(Rn, CHUNK_RAYS), raydist_mode_unit=opt.raydist_mode_unit)
    t_oracle = time.time() - t0
    n0 = int((pidx.clamp(min=0) == 0).sum())
    n_empty = int((pidx < 0).sum())
    err, conf0, untouched = step_errors(got, ref, keep, n0, point0_term(points["conf"], n_zo))
    # each ray colour within the forward's composite bound of float64 bounds the loss
    mse = float(((ts.last["out"]["coarse_raycolor"][0].cpu().double() - gt[hit].double()) ** 2).mean())
    d_loss, b_loss = abs(loss - loss64), loss_bound(loss, mse, fwd.BOUNDS["fp32" if precision == "fp32" else "general"]["composite"])
    pts_keys, mlp_keys = list(POINT_KEYS), [k for k in err if k not in POINT_KEYS]
    max_idx = int(keep.max())
    del net, npn, ts, got, q, kw, ex      # the next case gets the device without this one's 5M rows
    torch.cuda.empty_cache()
    print("\n[bench-f64] train %s F=%d mode=%d %s x%d: N=%d R'=%d of %d (hit %.3f) P=%d (%.1f x 2048) U=%d max point %d, empty slots %d (n0=%d) "
          "peak %.2f GB oracle %.0f s | points=%.2e (%s) mlp=%.2e (%s, %d tensors) conf0=%.2e/%.2e untouched=%s loss=%.9f |d|=%.2e/%.2e" % (
              cfg_name, F, mode, precision, batches, N, Rn, n_rays, Rn / n_rays, P, P / 2048, keep.numel(), max_idx, n_empty, n0, peak / 1e9, t_oracle,
              max(err[k] for k in pts_keys), max(pts_keys, key=err.get), max(err[k] for k in mlp_keys), max(mlp_keys, key=err.get),
              len(mlp_keys), conf0[0], conf0[1], untouched, loss, d_loss, b_loss))
    assert len(mlp_keys) == 18
    check_step(err, conf0, untouched, _rtol(mode, precision))
    assert d_loss <= b_loss, "loss %.9f vs float64 %.9f: %.3e > %.3e" % (loss, loss64, d_loss, b_loss)
    # the regime each case claims
    if cfg_name == "scannet_8gpu":
        assert max_idx >= 1 << 22, "no touched point above 2^22"
        assert Rn == n_rays, "a ray from inside the box misses its walls"
        if batches == 2:
            assert P > 64 * 2048, "%d pair rows: the split-K cap is not reached" % P
    else:
        assert 0.2 < Rn / n_rays < 0.8, "hit-ray fraction %.3f" % (Rn / n_rays)
    assert n_empty > 0


# ---- B. the forward, sample by sample, on the big frames; C. the whole frame equals its subsets ----
PRE_ROWS = 1 << 18          # rows of `pre` per float64 chunk


def _pre_errors_in_chunks(net, F):
    """test_gpu_forward_f64._pre_errors one chunk of rows at a time: every row of the hoisted table against float64
    b1 + W1[:, :7F] [f, PE3(f)], relative to the table's largest entry (in one piece it is an [N, 256] float64 matrix, 10 GB at 5M)."""
    npn = net.neural_points
    N = npn.xyz.shape[0]
    pre = net._pre[:N * 256].view(N, 256)
    emb = npn.points_embeding.detach()[0]
    w1 = net.aggregator.block1[0].weight.detach().cpu().double()[:, :7 * F]
    b1 = net.aggregator.block1[0].bias.detach().cpu().double()
    diff, scale = torch.empty(N, dtype=torch.float64), 0.0
    for i0 in range(0, N, PRE_ROWS):
        i1 = min(i0 + PRE_ROWS, N)
        f = emb[i0:i1].cpu().double()
        ref = b1 + torch.cat([f, shade_oracle.positional_encoding(f, 3)], dim=-1) @ w1.T
        diff[i0:i1] = (pre[i0:i1].cpu().double() - ref).abs().amax(-1)
        scale = max(scale, float(ref.abs().max()))
    return diff / scale


def frame_pixels(cfg, n=1024, seed=0):
    """n distinct pixels drawn from the whole frame (seeded), as (px, py)."""
    i = np.sort(np.random.RandomState(seed).choice(cfg.H * cfg.W, size=n, replace=False))
    return np.stack([i % cfg.W, i // cfg.W], -1).astype(np.float32)


def _block(x0, y0, w, h):
    px, py = np.meshgrid(np.arange(x0, x0 + w), np.arange(y0, y0 + h))
    return np.stack((px, py), -1).reshape(-1, 2).astype(np.float32)


TRUCK_CORNER = (860, 0, 100, 16)    # tests/test_gpu_shade.py: the limb crosses the strip (kernel_size 5)


@pytest.mark.parametrize("kernel", ["frozen", "general", "fp32"])
@pytest.mark.parametrize("cfg_name", ["truck_8gpu", "scannet_8gpu", "lego_render"])
def test_forward_over_the_whole_frame(cfg_name, kernel, monkeypatch):
    """B: _run on 1024 seeded pixels over the frame (truck: and the corner strip), the bench's camera; C: render_image of the whole
    frame equals render_full on those pixels, which equals forward()'s result on the hit rays, bit for bit."""
    monkeypatch.setattr(fwd, "_pre_errors", _pre_errors_in_chunks)
    with _device_released():
        _frame_case(cfg_name, kernel)


# the other bench lines on lego_render: bench_feat63.bench_render's 63-channel frame (F 63), bench_rw2c's per-point frames
# (scene.edit_frames, as test_gpu_forward_f64._run(frames=True) forms them)
LEGS = {"F63": dict(F=63), "rw2c": dict(frames=True)}


@pytest.mark.parametrize("kernel", ["frozen", "general", "fp32"])
@pytest.mark.parametrize("leg", list(LEGS))
def test_forward_over_the_whole_frame_bench_legs(leg, kernel, monkeypatch):
    """test_forward_over_the_whole_frame on lego_render for the bench_feat63 and bench_rw2c legs."""
    monkeypatch.setattr(fwd, "_pre_errors", _pre_errors_in_chunks)
    with _device_released():
        _frame_case("lego_render", kernel, **LEGS[leg])


def _frame_case(cfg_name, kernel, F=32, frames=False):
    cfg = scene.CONFIGS[cfg_name]
    pixels = frame_pixels(cfg)
    if cfg_name == "truck_8gpu":
        pixels = np.concatenate([pixels, _block(*TRUCK_CORNER)])
    _reset_peak_memory()
    net, sh, smap = fwd._run(cfg_name, F=F, kernel=kernel, frames=frames, rotated=False, pixels=pixels)
    hit, rays, out = smap["hit"], smap["rays"], smap["out"]
    pidx = smap["sample_pidx"]
    max_idx = int(pidx.max())
    cam, near, far, bg = rays["camrotc2w"][0], cfg.near, cfg.far, rays["bg_color"][0].tolist()
    with torch.no_grad():
        sub = net.render_full(rays["campos"][0].tolist(), rays["raydir"].to(DEV), cam, near, far, bg)
        frame = scene.make_rays(cfg)
        data = dict(frame, raydir=frame["raydir"].to(DEV))
        img = runner.render_image(net, data, cfg.H, cfg.W)
    net.check_errors()
    flat = torch.from_numpy((pixels[:, 1] * cfg.W + pixels[:, 0]).astype(np.int64)).to(DEV)
    same_sub = {k: torch.equal(sub[k][0][hit.to(DEV)], out[k][0]) for k in ("coarse_raycolor", "coarse_point_opacity", "coarse_is_background")}
    same_frame = {k: torch.equal(img[k].reshape(cfg.H * cfg.W, -1)[flat], sub[k][0].reshape(flat.shape[0], -1))
                  for k in ("coarse_raycolor", "coarse_point_opacity", "coarse_is_background", "ray_mask")}
    n_frame_hit = int(img["ray_mask"].sum())
    peak = torch.cuda.max_memory_allocated(DEV)
    del net, sub, img, out, smap
    torch.cuda.empty_cache()
    print("[bench-f64] frame %s F=%d frames=%s %s: %d pixels, %d hit; frame %dx%d, %d hit; max point %d; peak %.2f GB; subset == forward %s; "
          "frame == subset %s" % (cfg_name, F, frames, kernel, pixels.shape[0], int(hit.sum()), cfg.W, cfg.H, n_frame_hit, max_idx, peak / 1e9,
                                  same_sub, same_frame))
    assert all(same_sub.values()), "render_full on the subset differs from forward(): %s" % same_sub
    assert all(same_frame.values()), "the whole frame differs from render_full on its pixels: %s" % same_frame
    assert int(hit.sum()) > 200, "too few hit rays"
    if cfg_name == "scannet_8gpu":
        assert bool(hit.all()), "a ray inside the box misses its walls"
        if kernel == "frozen":
            assert max_idx >= 1 << 22, "no gathered point above 2^22: no pre row beyond 2^32 bytes"
