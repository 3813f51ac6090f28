"""Render cost of per-point frames (neural_points.Rw2c [N,3,3], edited / composed scenes) on the lego render workload of bench.py.

    python bench_rw2c.py --steps 20 --warmup 3 --rounds 3

One module, one full 800 x 800 frame per step (render_full, frozen-cloud pipeline).  Each round times the frame with the uniform
identity Rw2c and then with the two-object per-point frames of scene.edit_frames (cloud split by sign(x), each half in its own
rotation), so the two variants alternate within one process.  Per step the L2 is flushed, as in bench.py.  Prints one JSON line with
the card name and power limit next to the numbers.  Writes nothing.
"""
import argparse
import json
import statistics
import subprocess

import torch

from pointnerf_b200 import harness, scene


def card():
    name = torch.cuda.get_device_name()
    try:
        r = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader",
                            "-i", str(torch.cuda.current_device())], capture_output=True, text=True, timeout=30)
        smi = r.stdout.strip()
    except (OSError, subprocess.SubprocessError):
        smi = "nvidia-smi unavailable"
    return name, smi


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--steps", type=int, default=20)
    ap.add_argument("--warmup", type=int, default=3)
    ap.add_argument("--rounds", type=int, default=3)
    ap.add_argument("--precision", type=str, default="bf16x3")
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise RuntimeError("bench_rw2c.py needs a CUDA device: the product has no CPU path")
    dev = torch.device("cuda", 0)
    cfg = scene.CONFIGS["lego_render"]
    net, pts, opt = harness.build_model(cfg, dev, seed=0, alpha_bias=3.0, pnb_precision=args.precision)
    npn = net.neural_points
    frames = {"uniform": torch.eye(3, device=dev), "per_point": scene.edit_frames(pts["xyz"]).to(dev)}
    rays = scene.make_rays(cfg)["raydir"].to(dev)
    R = rays.shape[1]
    cam = (list(cfg.campos), torch.eye(3), cfg.near, cfg.far, [1., 1., 1.])
    flush = torch.empty(160 << 20, dtype=torch.uint8, device=dev)
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)

    def frame():
        with torch.no_grad():
            return net.render_full(cam[0], rays, cam[1], cam[2], cam[3], cam[4])

    def timed(kind):
        npn.Rw2c = frames[kind]                 # read in place by the kernels (per point) or by value (uniform)
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

    ms = {k: [] for k in frames}
    for _ in range(args.rounds):
        for kind in frames:
            ms[kind].append(timed(kind))
    cols = {}
    for kind in frames:
        npn.Rw2c = frames[kind]
        cols[kind] = frame()["coarse_raycolor"].clone()
    name, smi = card()
    res = dict(metric="lego render, uniform vs per-point Rw2c", gpu=name, nvidia_smi_name_power_limit=smi, precision=args.precision,
               rays_per_frame=R, steps=args.steps, rounds=args.rounds,
               ms_per_frame={k: [round(v, 4) for v in ms[k]] for k in ms},
               mrays_per_s_median={k: round(R / statistics.median(ms[k]) / 1e3, 3) for k in ms},
               per_point_over_uniform=round(statistics.median(ms["per_point"]) / statistics.median(ms["uniform"]), 4),
               max_abs_colour_change=float((cols["per_point"] - cols["uniform"]).abs().max()))
    print(json.dumps(res))


if __name__ == "__main__":
    main()
