"""Voxel down-sampling of the initial point cloud (run/train_ft.py:139, :690): construct_vox_points_closest of
pointnerf_b200.voxelize against the reference expression of models/mvs/mvs_utils.py:537-561 with torch_scatter's two calls written
as torch.Tensor.scatter_reduce_ ("mean", then "amin" and the lowest index among the minima).

    python bench_voxelize.py --steps 3 --warmup 1 --rounds 3

Workload: a synthetic scanned surface (a wavy ground sheet, a box's faces, 5% outliers) of 10M and 80M points at vox_res 320 and 800
(36 of the shipped scripts set vox_res in 320-900; train_ft.py caps the cloud at 80M points).  Each round times both legs, so they
alternate within one process; every timed window ends in a device synchronisation.  Peak memory: torch.cuda.max_memory_allocated over
one call of each leg, minus what was allocated before (the cloud).  Also reported: whether sparse_grid_idx is equal and the share of
voxels whose chosen point is the same (the reference's scatter order decides near-ties).
Prints one JSON line with the card name and power limit next to the numbers.  Writes nothing.
"""
import argparse
import json
import statistics
import subprocess

import torch

from pointnerf_b200 import voxelize


def card():
    name = torch.cuda.get_device_name()
    try:
        r = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader",
                            "-i", str(torch.cuda.current_device())], capture_output=True, text=True, timeout=30)
        smi = r.stdout.strip()
    except (OSError, subprocess.SubprocessError):
        smi = "nvidia-smi unavailable"
    return name, smi


def surface(n, dev, seed=0):
    g = torch.Generator(device=dev).manual_seed(seed)
    n1, n2 = n * 6 // 10, n * 35 // 100
    uv = torch.rand((n1, 2), generator=g, device=dev)
    ground = torch.stack([uv[:, 0] * 8 - 4, uv[:, 1] * 8 - 4, 0.2 * torch.sin(3 * uv[:, 0]) * torch.cos(2 * uv[:, 1])], 1)
    w = torch.rand((n2, 3), generator=g, device=dev) * 2 - 1
    f = torch.randint(0, 6, (n2,), generator=g, device=dev)
    w[torch.arange(n2, device=dev), f // 2] = torch.where(f % 2 == 1, 1.0, -1.0)
    box = w * torch.tensor([1.0, 0.7, 0.5], device=dev) + torch.tensor([0.5, -0.3, 0.6], device=dev)
    out = torch.rand((n - n1 - n2, 3), generator=g, device=dev) * 12 - 6
    return torch.cat([ground, box, out]).contiguous()


def reference_closest(xyz_val, vox_res):
    """mvs_utils.py:537-561 (space_min None) with scatter_mean / scatter_min on scatter_reduce_."""
    xyz = xyz_val
    xyz_min, xyz_max = torch.min(xyz, dim=-2)[0], torch.max(xyz, dim=-2)[0]
    space_edge = torch.max(xyz_max - xyz_min) * 1.05
    xyz_mid = (xyz_max + xyz_min) / 2
    space_min = xyz_mid - space_edge / 2
    construct_vox_sz = space_edge / vox_res
    xyz_shift = xyz - space_min[None, ...]
    sparse_grid_idx, inv_idx = torch.unique(torch.floor(xyz_shift / construct_vox_sz[None, ...]).to(torch.int32), dim=0, return_inverse=True)
    m = sparse_grid_idx.shape[0]
    xyz_centroid = torch.zeros((m, 3), device=xyz.device).scatter_reduce_(0, inv_idx[:, None].expand(-1, 3), xyz_val, "mean",
                                                                          include_self=False)
    xyz_residual = torch.norm(xyz_val - xyz_centroid[inv_idx, :], dim=-1)
    rmin = torch.zeros(m, device=xyz.device).scatter_reduce_(0, inv_idx, xyz_residual, "amin", include_self=False)
    pos = torch.arange(xyz.shape[0], device=xyz.device)
    hit = xyz_residual == rmin[inv_idx]
    min_idx = torch.full((m,), xyz.shape[0], device=xyz.device).scatter_reduce_(0, inv_idx[hit], pos[hit], "amin")
    return xyz_centroid, sparse_grid_idx, min_idx


LEGS = {"fused": voxelize.construct_vox_points_closest, "reference_expr": reference_closest}


def bench_case(args, dev, n, vox_res):
    xyz = surface(n, dev)
    torch.cuda.synchronize(dev)
    peak, outs = {}, {}
    for leg, fn in LEGS.items():
        torch.cuda.empty_cache()
        torch.cuda.synchronize(dev)
        base = torch.cuda.memory_allocated(dev)
        torch.cuda.reset_peak_memory_stats(dev)
        outs[leg] = fn(xyz, vox_res)
        torch.cuda.synchronize(dev)
        peak[leg] = (torch.cuda.max_memory_allocated(dev) - base) / 2 ** 20
    a, b = outs["fused"], outs["reference_expr"]
    grid_equal = torch.equal(a[1], b[1])
    same_point = float((a[2] == b[2]).float().mean()) if grid_equal else None
    cen_max_abs = float((a[0] - b[0]).abs().max()) if grid_equal else None
    m = a[1].shape[0]
    del outs, a, b
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    ms = {leg: [] for leg in LEGS}
    for _ in range(args.rounds):
        for leg, fn in LEGS.items():
            for _ in range(args.warmup):
                fn(xyz, vox_res)
            torch.cuda.synchronize(dev)
            e0.record()
            for _ in range(args.steps):
                fn(xyz, vox_res)
            e1.record()
            torch.cuda.synchronize(dev)
            ms[leg].append(e0.elapsed_time(e1) / args.steps)
    del xyz
    torch.cuda.empty_cache()
    med = {leg: statistics.median(v) for leg, v in ms.items()}
    return dict(points=n, vox_res=vox_res, voxels=m, ms_per_call_median={k: round(v, 2) for k, v in med.items()},
                ms_per_call_min_max={k: [round(min(v), 2), round(max(v), 2)] for k, v in ms.items()},
                peak_mb_over_cloud={k: round(v, 1) for k, v in peak.items()},
                reference_over_fused=round(med["reference_expr"] / med["fused"], 2), sparse_grid_idx_equal=grid_equal,
                same_closest_point_share=same_point, centroid_max_abs_diff=cen_max_abs)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--steps", type=int, default=3)
    ap.add_argument("--warmup", type=int, default=1)
    ap.add_argument("--rounds", type=int, default=3)
    ap.add_argument("--points", type=int, nargs="+", default=[10_000_000, 80_000_000])
    ap.add_argument("--vox_res", type=float, nargs="+", default=[320, 800])
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise RuntimeError("bench_voxelize.py needs a CUDA device: the product has no CPU path")
    dev = torch.device("cuda", 0)
    res = [bench_case(args, dev, n, r) for n in args.points for r in args.vox_res]
    name, smi = card()
    print(json.dumps(dict(metric="construct_vox_points_closest on a synthetic surface: fused vs the reference expression "
                                 "(torch.unique + scatter_reduce_)", gpu=name, nvidia_smi_name_power_limit=smi, steps=args.steps,
                          warmup=args.warmup, rounds=args.rounds, cases=res)))


if __name__ == "__main__":
    main()
