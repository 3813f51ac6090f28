"""Probe pass of point growing (opt.prob = 1) over whole training frames: runner.probe_image (one call per frame, k_probe_outputs
on the full-R query) against probe_hole's pattern (run/train_ft.py:417-530: 2304-ray chunks through forward(), assembled into
[H, W, C] maps; runner.probe_image_chunked).

    python bench_probe.py --steps 3 --warmup 1 --rounds 3

Workload: the lego 800 x 800 frame (N = 400k, bench.py's lego_render scene) at SR 24 and at SR 80 (the NeRF-synthetic scripts).  Each
round times both legs, so they alternate within one process; every timed window ends in a device synchronisation.  Peak memory:
torch.cuda.max_memory_allocated over one frame of each leg on its own module, minus what was allocated before (points, MLP).
The parent commit's eager probe (dense export + torch ops per chunk) is not timed here.
Prints one JSON line with the card name and power limit next to the numbers.  Writes nothing.
"""
import argparse
import json
import statistics
import subprocess

import torch

from pointnerf_b200 import harness, runner, scene


def card():
    name = torch.cuda.get_device_name()
    try:
        r = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader",
                            "-i", str(torch.cuda.current_device())], capture_output=True, text=True, timeout=30)
        smi = r.stdout.strip()
    except (OSError, subprocess.SubprocessError):
        smi = "nvidia-smi unavailable"
    return name, smi


LEGS = ("whole_frame", "chunked_2304")


def _leg(name, net, data, cfg):
    if name == "whole_frame":
        return runner.probe_image(net, data, cfg.H, cfg.W)
    return runner.probe_image_chunked(net, data, cfg.H, cfg.W, 2304)


def bench_sr(args, dev, SR):
    cfg = scene.CONFIGS["lego_render"]
    rays = scene.make_rays(cfg)
    data = {k: (v.to(dev) if isinstance(v, torch.Tensor) else v) for k, v in rays.items()}
    build = lambda: harness.build_model(cfg, dev, seed=0, alpha_bias=3.0, SR=SR, prob=1)[0]
    # peak memory of one frame per leg, each on its own module
    peak = {}
    for leg in LEGS:
        torch.cuda.empty_cache()
        net = build()
        torch.cuda.synchronize(dev)
        base = torch.cuda.memory_allocated(dev)
        torch.cuda.reset_peak_memory_stats(dev)
        _leg(leg, net, data, cfg)
        torch.cuda.synchronize(dev)
        peak[leg] = (torch.cuda.max_memory_allocated(dev) - base) / 2 ** 20
        del net
    nets = {leg: build() for leg in LEGS}
    same = all(torch.equal(a, b) for a, b in zip(_leg(LEGS[0], nets[LEGS[0]], data, cfg).values(),
                                                _leg(LEGS[1], nets[LEGS[1]], data, cfg).values()))
    hit = None
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    ms = {leg: [] for leg in LEGS}
    for _ in range(args.rounds):
        for leg, net in nets.items():
            for _ in range(args.warmup):
                m = _leg(leg, net, data, cfg)
            torch.cuda.synchronize(dev)
            e0.record()
            for _ in range(args.steps):
                m = _leg(leg, net, data, cfg)
            e1.record()
            torch.cuda.synchronize(dev)
            net.check_errors()
            ms[leg].append(e0.elapsed_time(e1) / args.steps)
            hit = int((m["ray_mask"] > 0).sum())
    del nets
    torch.cuda.empty_cache()
    med = {leg: statistics.median(v) for leg, v in ms.items()}
    return dict(rays=cfg.H * cfg.W, hit_rays=hit, ms_per_frame_median={k: round(v, 3) for k, v in med.items()},
                ms_per_frame_min_max={k: [round(min(v), 3), round(max(v), 3)] for k, v in ms.items()},
                peak_mb_over_model={k: round(v, 1) for k, v in peak.items()},
                chunked_over_whole=round(med[LEGS[1]] / med[LEGS[0]], 2), maps_bit_identical=same)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--steps", type=int, default=3)
    ap.add_argument("--warmup", type=int, default=1)
    ap.add_argument("--rounds", type=int, default=3)
    ap.add_argument("--sr", type=int, nargs="+", default=[24, 80])
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise RuntimeError("bench_probe.py needs a CUDA device: the product has no CPU path")
    dev = torch.device("cuda", 0)
    res = {"SR%d" % sr: bench_sr(args, dev, sr) for sr in args.sr}
    name, smi = card()
    print(json.dumps(dict(metric="probe pass of one lego 800x800 training frame: probe_image vs 2304-ray chunks through forward()",
                          gpu=name, nvidia_smi_name_power_limit=smi, steps=args.steps, warmup=args.warmup, rounds=args.rounds,
                          parent_eager_probe="not measured", **res)))


if __name__ == "__main__":
    main()
