"""Query-only throughput of this project's perspective-frustum query (wcoord_query 0, NN 2; pointnerf_b200.query_point_indices) on a
DTU-sized view: one full-frame call, and the same querier driven the way the reference's test loop drives a querier, 2304-ray chunks
over the view (one build, reused).  Neither number times the reference's own kernels.  Each figure is the median of --rounds timed
windows of --reps repetitions, with the min and max beside it; the card's name and power limit are printed with the numbers.

A second line times the fused module on the same query (pointnerf_b200.ray_marching with wcoord_query 0, the DTU scripts' F = 63
and point modes 01): the whole-frame render of the view through runner.render_image (query, shading and compositing, fill_invalid in
the kernel, one host synchronisation for R' and one for the frame's status), and one training step on a 48x48-ray patch (forward with
jitter, colour + zero_one loss, backward).  The two legs alternate inside every round, in one process.

    python bench_frustum.py [--rounds 5] [--reps 100] [--chunk-reps 5] [--warmup 3] [--fused-reps 5]
"""
import argparse
import json
import subprocess
import time

import numpy as np
import torch

from pointnerf_b200 import harness, runner, scene
from pointnerf_b200 import query_point_indices as qpi
from pointnerf_b200.ray_marching import NeuralPoints, NeuralPointsRayMarching, PointAggregator


def card():
    try:
        out = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"], capture_output=True,
                             text=True, timeout=30).stdout.strip().splitlines()[0]
        return [v.strip() for v in out.split(",")]
    except Exception:  # noqa: BLE001
        return [torch.cuda.get_device_name(0), "unknown", "unknown"]


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--rounds", type=int, default=5)
    ap.add_argument("--reps", type=int, default=100)        # full-frame calls per window (~0.6 s)
    ap.add_argument("--chunk-reps", type=int, default=5)    # chunk loops per window (~0.5 s)
    ap.add_argument("--warmup", type=int, default=3)
    ap.add_argument("--fused-reps", type=int, default=5)    # frames / training steps per window of the fused legs
    a = ap.parse_args()
    assert torch.cuda.is_available(), "bench_frustum.py needs a GPU"
    dev = torch.device("cuda:0")
    # the DTU scripts' frame (800 x 600) and query options, a 400k-point surface
    cfg = scene.FrustumConfig("dtu_frame", N=400_000, H=600, W=800, focal=1000.0)
    s = scene.make_frustum_scene(cfg)
    opt = scene.frustum_opt(cfg)
    q = qpi.lighting_fast_querier(dev, opt)
    pers = torch.from_numpy(s["pers"]).to(dev)[None]
    xyz_w = torch.from_numpy(s["xyz_w"]).to(dev)[None]
    camrot = torch.from_numpy(s["camrotc2w"]).to(dev)[None]
    campos = torch.from_numpy(s["campos"]).to(dev)[None]
    npts = torch.tensor([cfg.N], dtype=torch.int32, device=dev)
    pix = torch.from_numpy(s["pixel_idx"]).to(dev)[None]
    R = pix.shape[1]

    def run(p):
        return q.query_points(p, pers, xyz_w, npts, np.int64(cfg.H), np.int64(cfg.W), s["intrinsic"], np.float32(cfg.near),
                              np.float32(cfg.far), None, campos, camrot)

    def timed(fn, reps):
        """Median, min and max over the rounds of the mean time per repetition (ms)."""
        for _ in range(a.warmup):
            fn()
        torch.cuda.synchronize()
        ts = []
        for _ in range(a.rounds):
            t0 = time.perf_counter()
            for _ in range(reps):
                fn()
            torch.cuda.synchronize()
            ts.append((time.perf_counter() - t0) / reps * 1e3)
        return dict(median_ms=round(float(np.median(ts)), 3), min_ms=round(min(ts), 3), max_ms=round(max(ts), 3))

    kept = run(pix)[0].shape[1]
    full = timed(lambda: run(pix), a.reps)
    n_chunks = (R + 2303) // 2304
    builds = q.n_builds
    chunks = timed(lambda: [run(pix[:, k:k + 2304]) for k in range(0, R, 2304)], a.chunk_reps)
    assert q.n_builds == builds, "the chunk loop must reuse the view's build"
    rebuild = timed(lambda: (q.clean_up(), run(pix[:, :2304])), a.reps)
    name, power, clk = card()
    print(json.dumps(dict(metric="frustum_query (this project's querier)", gpu=name, power_limit=power, max_sm_clock=clk, rays=R,
                          points=cfg.N, kept_rays_full_frame=int(kept), full_frame=full,
                          full_frame_mrays_s=round(R / full["median_ms"] / 1e3, 2), chunk_loop=chunks, chunks=n_chunks,
                          chunk_loop_mrays_s=round(R / chunks["median_ms"] / 1e3, 2), build_plus_one_chunk=rebuild,
                          rounds=a.rounds, reps=a.reps, chunk_reps=a.chunk_reps)))
    fused(a, dev, cfg, s, pix, name, power, clk)


def fused_net(dev, cfg, s, is_train):
    """The fused module on the frustum view: the DTU scripts' options, the scene's 63-channel points, an opaque surface."""
    opt = harness.make_opt(scene.CONFIGS["tiny"], feat_dim=63, **vars(scene.frustum_opt(cfg, is_train=is_train)))
    pts = scene.make_frustum_points(cfg, s)
    agg = PointAggregator(opt, seed=5)
    with torch.no_grad():
        agg.alpha_branch[0].bias += 300.0
    npn = NeuralPoints(opt, dev)
    npn.set_points(pts["xyz"].to(dev), pts["embedding"].to(dev), points_color=pts["color"].to(dev), points_dir=pts["dir"].to(dev),
                   points_conf=pts["conf"].to(dev), parameter=True, as_stored=True)
    return NeuralPointsRayMarching(aggregator=agg.to(dev), neural_points=npn, opt=opt)


def fused(a, dev, cfg, s, pix, name, power, clk):
    R = pix.shape[1]
    data = dict(campos=torch.from_numpy(s["campos"]).to(dev)[None], camrotc2w=torch.from_numpy(s["camrotc2w"]).to(dev)[None],
                raydir=torch.zeros((1, R, 3), device=dev), pixel_idx=pix, h=cfg.H, w=cfg.W, intrinsic=s["intrinsic"], near=cfg.near,
                far=cfg.far, bg_color=torch.ones(3, device=dev))
    render_net = fused_net(dev, cfg, s, False)
    train_net = fused_net(dev, cfg, s, True)
    # the training patch: 48 x 48 pixels around the centre of the frame (random_sample_size 48)
    y0, x0 = cfg.H // 2 - 24, cfg.W // 2 - 24
    py, px = np.meshgrid(np.arange(y0, y0 + 48), np.arange(x0, x0 + 48), indexing="ij")
    patch = torch.from_numpy(np.stack([px, py], -1).reshape(1, -1, 2).astype(np.int32)).to(dev)
    gt = torch.rand((1, 48 * 48, 3), device=dev)
    npn = train_net.neural_points
    params = list(train_net.aggregator.parameters()) + [npn.points_embeding, npn.points_color, npn.points_dir, npn.points_conf]

    def frame():
        return runner.render_image(render_net, data, cfg.H, cfg.W)

    def step():
        for p in params:
            p.grad = None
        out = train_net(data["campos"], data["raydir"][:, :48 * 48], bg_color=data["bg_color"], camrotc2w=data["camrotc2w"],
                        pixel_idx=patch, near=cfg.near, far=cfg.far, h=cfg.H, w=cfg.W, intrinsic=s["intrinsic"])
        hit = torch.nonzero(out["ray_mask"][0])[:, 0]
        cc = torch.clamp(out["conf_coefficient"], 1e-3, 1 - 1e-3)
        loss = ((out["coarse_raycolor"][0] - gt[0][hit]) ** 2).mean() + 1e-3 * torch.mean(torch.log(cc) + torch.log(1 - cc))
        loss.backward()

    for _ in range(a.warmup):
        frame()
        step()
    torch.cuda.synchronize()
    ts = dict(frame=[], step=[])
    for _ in range(a.rounds):                      # the two legs alternate inside every round
        for leg, fn in (("frame", frame), ("step", step)):
            torch.cuda.synchronize()
            t0 = time.perf_counter()
            for _ in range(a.fused_reps):
                fn()
            torch.cuda.synchronize()
            ts[leg].append((time.perf_counter() - t0) / a.fused_reps * 1e3)
    render_net.check_errors()
    train_net.check_errors()
    summ = {k: dict(median_ms=round(float(np.median(v)), 3), min_ms=round(min(v), 3), max_ms=round(max(v), 3)) for k, v in ts.items()}
    print(json.dumps(dict(metric="frustum_fused (render_image of the view; 48x48-ray training step)", gpu=name, power_limit=power,
                          max_sm_clock=clk, rays=R, points=cfg.N, whole_frame=summ["frame"],
                          whole_frame_mrays_s=round(R / summ["frame"]["median_ms"] / 1e3, 2), train_step_48x48=summ["step"],
                          train_steps_s=round(1e3 / summ["step"]["median_ms"], 1), rounds=a.rounds, reps=a.fused_reps)))


if __name__ == "__main__":
    main()
