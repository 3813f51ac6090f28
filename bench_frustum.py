"""Query-only throughput of this project's perspective-frustum query (wcoord_query 0, NN 2; pointnerf_b200.query_point_indices) on a
DTU-sized view: one full-frame call, and the same querier driven the way the reference's test loop drives a querier, 2304-ray chunks
over the view (one build, reused).  Neither number times the reference's own kernels.  Each figure is the median of --rounds timed
windows of --reps repetitions, with the min and max beside it; the card's name and power limit are printed with the numbers.

    python bench_frustum.py [--rounds 5] [--reps 100] [--chunk-reps 5] [--warmup 3]
"""
import argparse
import json
import subprocess
import time

import numpy as np
import torch

from pointnerf_b200 import query_point_indices as qpi
from pointnerf_b200 import scene


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


if __name__ == "__main__":
    main()
