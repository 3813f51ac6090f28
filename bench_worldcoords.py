"""Cost of reading the query options on every call: the world-coordinate querier of wcoord_query 1
(pointnerf_b200.query_point_indices_worldcoords, options read from opt per call) against the wcoord_query -1 querier
(pointnerf_b200.point_query, options read once at construction), both driven the way the reference's loops drive a querier: query_points
on 2304-ray chunks over a whole lego-sized 800x800 view (400k points, SR 24, K 8), the grid built once and reused.  The two legs
alternate inside every round, in one process, and each figure is the median of --rounds timed windows with the min and max beside it,
as time per query_points call; the difference between the legs is taken round by round.  A third figure is the host time of the
per-call work that differs between the two (wcoord_query 1: the option read and the grid lookup keyed on the options; -1: the grid
lookup), on the cached grid, averaged over many calls.  Neither leg times the reference's own kernels.  The card's name and power limit
are printed with the numbers.

    python bench_worldcoords.py [--rounds 10] [--loops 2] [--warmup 1]
"""
import argparse
import json
import subprocess
import time

import numpy as np
import torch

from pointnerf_b200 import harness, scene
from pointnerf_b200 import point_query as wq
from pointnerf_b200 import query_point_indices_worldcoords as wc

CHUNK = 2304


def card():
    try:
        out = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"], capture_output=True,
                             text=True, timeout=30).stdout.strip().splitlines()[0]
        return [v.strip() for v in out.split(",")]
    except Exception:  # noqa: BLE001
        return [torch.cuda.get_device_name(0), "unknown", "unknown"]


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--rounds", type=int, default=10)
    ap.add_argument("--loops", type=int, default=2)          # chunk loops over the view per leg and window
    ap.add_argument("--warmup", type=int, default=1)
    a = ap.parse_args()
    assert torch.cuda.is_available(), "bench_worldcoords.py needs a GPU"
    dev = torch.device("cuda:0")
    cfg = scene.CONFIGS["lego_render"]
    xyz = scene.make_points(cfg)["xyz"].to(dev).contiguous()
    r = {k: (v.to(dev) if isinstance(v, torch.Tensor) else v) for k, v in scene.make_rays(cfg).items()}
    R = r["raydir"].shape[1]
    pix = r["pixel_idx"].to(torch.int32)
    near, far = np.float32(r["near"].item()), np.float32(r["far"].item())
    queriers = {"wcoord_query_-1": wq.lighting_fast_querier(dev, harness.make_opt(cfg)),
                "wcoord_query_1": wc.lighting_fast_querier(dev, harness.make_opt(cfg, wcoord_query=1))}

    def loop(q):
        hits = 0
        for k in range(0, R, CHUNK):
            out = q.query_points(pix[:, k:k + CHUNK], None, xyz[None], None, 0, 0, None, near, far, r["raydir"][:, k:k + CHUNK],
                                 r["campos"], r["camrotc2w"])
            hits += out[0].shape[1]
        return hits

    hits = {}
    for name, q in queriers.items():
        for _ in range(a.warmup):
            hits[name] = loop(q)
    assert hits["wcoord_query_-1"] == hits["wcoord_query_1"] > 0
    torch.cuda.synchronize()
    n_calls = (R + CHUNK - 1) // CHUNK
    ts = {name: [] for name in queriers}
    names = list(queriers)
    for i in range(a.rounds):                     # the two legs alternate inside every round, first one and then the other leading
        for name in (names if i % 2 == 0 else names[::-1]):
            torch.cuda.synchronize()
            t0 = time.perf_counter()
            for _ in range(a.loops):
                loop(queriers[name])
            torch.cuda.synchronize()
            ts[name].append((time.perf_counter() - t0) / (a.loops * n_calls) * 1e6)
    assert all(q.n_builds == 1 for q in queriers.values()), "the chunk loops must reuse one grid build"
    # the host work that differs between the two per call: the option read and the grid lookup (with the key on the options) of
    # wcoord_query 1 against the grid lookup of -1, on the cached grid
    q_1, q1 = queriers["wcoord_query_-1"], queriers["wcoord_query_1"]
    host = {}
    for name, fn in (("wcoord_query_-1", lambda: q_1._grid_for(xyz)), ("wcoord_query_1", lambda: (q1._read_options(), q1._grid_for(xyz)))):
        reps = 20000
        t0 = time.perf_counter()
        for _ in range(reps):
            fn()
        host[name] = (time.perf_counter() - t0) / reps * 1e6
    diffs = [b - a_ for a_, b in zip(ts["wcoord_query_-1"], ts["wcoord_query_1"])]
    summ = {k: dict(median_us=round(float(np.median(v)), 1), min_us=round(min(v), 1), max_us=round(max(v), 1)) for k, v in ts.items()}
    name, power, clk = card()
    print(json.dumps(dict(metric="query_points per 2304-ray call over an 800x800 view (lego_render: 400k points, SR 24, K 8)", gpu=name,
                          power_limit=power, max_sm_clock=clk, rays=R, calls_per_view=n_calls, hit_rays=int(hits["wcoord_query_1"]),
                          per_call=summ, difference_us=dict(median=round(float(np.median(diffs)), 1), min=round(min(diffs), 1),
                                                            max=round(max(diffs), 1)),
                          host_lookup_us={k: round(v, 2) for k, v in host.items()}, rounds=a.rounds, loops=a.loops)))


if __name__ == "__main__":
    main()
