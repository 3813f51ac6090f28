"""Cost of the DTU point width (point_features_dim 63, point_{conf,dir,color}_mode "01") against the usual 32 channels.

    python bench_feat63.py --steps 20 --warmup 3 --rounds 3

render: the lego render workload of bench.py (one full 800 x 800 frame per step, render_full, frozen-cloud pipeline) with a 32- and a
63-channel cloud of the same points; each round times both, so the two widths alternate within one process.  Per step the L2 is
flushed, as in bench.py.
train: a ship_optimise-sized optimisation step (N = 600k, 3600 random rays of one view, forward + backward + 2x Adam through
parallel.TrainStep on one rank) at both widths, alternating as well.
Prints one JSON line with the card name and power limit next to the numbers.  Writes nothing.
"""
import argparse
import json
import statistics
import subprocess

import numpy as np
import torch

from pointnerf_b200 import harness, parallel, scene


def card():
    name = torch.cuda.get_device_name()
    try:
        r = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader",
                            "-i", str(torch.cuda.current_device())], capture_output=True, text=True, timeout=30)
        smi = r.stdout.strip()
    except (OSError, subprocess.SubprocessError):
        smi = "nvidia-smi unavailable"
    return name, smi


def bench_render(args, dev):
    cfg = scene.CONFIGS["lego_render"]
    nets = {F: harness.build_model(cfg, dev, seed=0, alpha_bias=3.0, pnb_precision=args.precision, feat_dim=F)[0] for F in (32, 63)}
    rays = scene.make_rays(cfg)["raydir"].to(dev)
    R = rays.shape[1]
    cam = (list(cfg.campos), torch.eye(3), cfg.near, cfg.far, [1., 1., 1.])
    flush = torch.empty(160 << 20, dtype=torch.uint8, device=dev)
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)

    def timed(net):
        def frame():
            with torch.no_grad():
                return net.render_full(cam[0], rays, cam[1], cam[2], cam[3], cam[4])
        for _ in range(args.warmup):
            frame()
        net.check_errors()
        torch.cuda.synchronize(dev)
        e0.record()
        for _ in range(args.steps):
            flush.fill_(1)
            frame()
        e1.record()
        torch.cuda.synchronize(dev)
        net.check_errors()
        return e0.elapsed_time(e1) / args.steps

    ms = {F: [] for F in nets}
    for _ in range(args.rounds):
        for F, net in nets.items():
            ms[F].append(timed(net))
    del nets
    torch.cuda.empty_cache()
    return R, ms


def bench_train(args, dev):
    cfg = scene.CONFIGS["ship_optimise"]
    steps = {}
    for F in (32, 63):
        net = harness.build_model(cfg, dev, alpha_bias=3.0, is_train=True, pnb_precision=args.precision, feat_dim=F)[0]
        steps[F] = (net, parallel.TrainStep(net, world=1, rank=0))
    rng = np.random.RandomState(0)
    g = torch.Generator().manual_seed(1)

    def batch():
        px = rng.randint(0, cfg.W, size=(3600,)).astype(np.float32)
        py = rng.randint(0, cfg.H, size=(3600,)).astype(np.float32)
        gt = torch.rand(3600, 3, generator=g)
        rays = {k: (v.to(dev) if k in ("raydir", "pixel_idx") else v) for k, v in scene.make_rays(cfg, np.stack([px, py], -1)).items()}
        kw = dict(campos=rays["campos"], raydir=rays["raydir"], bg_color=rays["bg_color"], camrotc2w=rays["camrotc2w"], pixel_idx=rays["pixel_idx"],
                  near=rays["near"], far=rays["far"], h=rays["h"], w=rays["w"], intrinsic=rays["intrinsic"])
        return kw, gt.to(dev)

    batches = [batch() for _ in range(args.warmup + args.steps)]
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    ms = {F: [] for F in steps}
    for _ in range(args.rounds):
        for F, (net, ts) in steps.items():
            for kw, gt in batches[:args.warmup]:
                ts.step(kw, gt)
            torch.cuda.synchronize(dev)
            e0.record()
            for kw, gt in batches[args.warmup:]:
                ts.step(kw, gt)
            e1.record()
            torch.cuda.synchronize(dev)
            net.check_errors()
            ms[F].append(e0.elapsed_time(e1) / args.steps)
    return ms


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--steps", type=int, default=20)
    ap.add_argument("--warmup", type=int, default=3)
    ap.add_argument("--rounds", type=int, default=3)
    ap.add_argument("--precision", type=str, default="bf16x3")
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise RuntimeError("bench_feat63.py needs a CUDA device: the product has no CPU path")
    dev = torch.device("cuda", 0)
    R, rms = bench_render(args, dev)
    tms = bench_train(args, dev)
    name, smi = card()
    res = dict(metric="point_features_dim 32 vs 63: lego render, ship_optimise training step", gpu=name, nvidia_smi_name_power_limit=smi,
               precision=args.precision, rays_per_frame=R, steps=args.steps, rounds=args.rounds,
               render_ms_per_frame={F: [round(v, 4) for v in rms[F]] for F in rms},
               render_mrays_per_s_median={F: round(R / statistics.median(rms[F]) / 1e3, 3) for F in rms},
               render_63_over_32=round(statistics.median(rms[63]) / statistics.median(rms[32]), 4),
               train_ms_per_step={F: [round(v, 4) for v in tms[F]] for F in tms},
               train_steps_per_s_median={F: round(1e3 / statistics.median(tms[F]), 2) for F in tms},
               train_63_over_32=round(statistics.median(tms[63]) / statistics.median(tms[32]), 4))
    print(json.dumps(res))


if __name__ == "__main__":
    main()
