"""Benchmark of the initial point cloud's geometric steps: depth_filter.filter_by_masks_gpu at the DTU size (49 views, 512x640) and an
n360 size (100 views, 800x800), and depth_filter.alpha_masking at 10M and 50M points x 100 views, each against the reference
expression (filter_utils.filter_by_masks_gpu and mvs_utils.alpha_masking restated below in eager torch: per ordered view pair, the
projection, grid_sample and back-projection on full H x W temporaries; per view, the int64 pixel temporaries), alternating in one
process.  Prints one JSON line per case with both legs' times, peak memory, both legs' counts and whether they agree, and the card's
name and power limit; times are the median and range over --reps calls of each leg after one warm-up call.  The reference leg runs on the GPU with cuBLAS matmuls and fp32 inverses, so its counts can differ where a
decision sits within rounding of its threshold (tests/test_depth_filter_oracle.py bounds that difference).

python bench_depth_filter.py [--reps 3] [--only dtu,n360,alpha10m,alpha50m]
"""
import argparse
import json
import statistics
import os
import subprocess
import sys
import time
import types

import torch
import torch.nn.functional as Fn

sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, os.path.join(os.path.dirname(os.path.abspath(__file__)), "tests"))
from pointnerf_b200 import depth_filter  # noqa: E402


def ref_filter(cam_xyz_all, Ks, Es, confs, masks, opt):
    """The reference expression: for every ref view, every src view's reprojection test on whole-image tensors."""
    V = len(cam_xyz_all)
    H, W = cam_xyz_all[0].shape[3:5]
    dev = cam_xyz_all[0].device
    yy, xx = torch.meshgrid(torch.arange(H, device=dev), torch.arange(W, device=dev), indexing="ij")
    xx, yy = xx.reshape(-1), yy.reshape(-1)
    ones = torch.ones_like(xx)
    outs = []
    for r in range(V):
        xyz = cam_xyz_all[r][0, 0, 0]
        d = xyz[..., 2]
        Kr, Er = Ks[r][0], Es[r][0]
        geo, dsum = 0, 0
        pr = torch.linalg.inv(Kr) @ (torch.stack([xx, yy, ones]) * d.reshape(-1))
        for s in range(V):
            if s == r:
                continue
            Ks_, Es_ = Ks[s][0], Es[s][0]
            ps = (Es_ @ torch.linalg.inv(Er) @ torch.cat([pr, ones[None]]))[:3]
            k = Ks_ @ ps
            uv = k[:2] / k[2:3]
            gx, gy = uv[0].reshape(H, W), uv[1].reshape(H, W)
            grid = torch.stack([gx * 2 / (W - 1) - 1, gy * 2 / (H - 1) - 1], -1)[None]
            ds = Fn.grid_sample(cam_xyz_all[s][0, 0, 0][..., 2][None, None], grid, align_corners=True, mode="bilinear",
                                padding_mode="border").reshape(-1)
            q = torch.linalg.inv(Ks_) @ (torch.cat([uv, ones[None]]) * ds)
            e = (Er @ torch.linalg.inv(Es_) @ torch.cat([q, ones[None]]))[:3]
            dre = e[2].reshape(H, W)
            k2 = Kr @ e
            xr, yr = (k2[0] / k2[2]).reshape(H, W), (k2[1] / k2[2]).reshape(H, W)
            dist = torch.sqrt((xr - xx.reshape(H, W)) ** 2 + (yr - yy.reshape(H, W)) ** 2)
            m = (dist < 1) & ((dre - d).abs() / d < 0.01)
            dre = torch.where(m, dre, torch.zeros_like(dre))
            geo = geo + m.to(torch.int32)
            dsum = dsum + dre
        avg = (dsum + d) / (geo + 1)
        keep = (confs[r][0, 0] > opt.depth_conf_thresh) & masks[r][0, 0] & (geo >= opt.geo_cnsst_num)
        cam = torch.cat([xyz[..., :2][keep], avg[keep][..., None]], -1)
        world = (torch.cat([cam, torch.ones_like(cam[:, :1])], -1) @ torch.inverse(Er).t())[:, :3]
        rg = torch.as_tensor(opt.ranges, device=dev, dtype=torch.float32)
        inr = torch.all((world >= rg[:3]) & (world <= rg[3:]), -1)
        outs.append((cam[inr], world[inr], confs[r][0, 0][keep][inr]))
    return outs


def ref_alpha(points, alphas, Ks, w2cs, near_far):
    """The reference expression: per view, homogeneous [N,4] and [N,3] products and int64 pixel coordinates."""
    p1 = torch.cat([points, torch.ones_like(points[:, :1])], -1)
    H, W = alphas[0].shape
    out = None
    for a, K, w in zip(alphas, Ks, w2cs):
        cam = p1 @ w.t()
        nf = (cam[:, 2] >= near_far[0] - 1.0) & (cam[:, 2] <= near_far[1])
        k = cam[:, :3] @ K.t()
        ij = torch.floor(k[:, :2] / k[:, 2:]).long()
        inr = ((ij >= 0) & (ij < torch.tensor([[W, H]], device=ij.device))).all(-1)
        ij[:, 0].clamp_(0, W - 1)
        ij[:, 1].clamp_(0, H - 1)
        m = ((a[ij[:, 1], ij[:, 0]] + (~inr).float()) > 0.1) & nf
        out = m if out is None else out & m
    return out


def _timed(fn):
    torch.cuda.synchronize()
    torch.cuda.reset_peak_memory_stats()
    t = time.perf_counter()
    r = fn()
    torch.cuda.synchronize()
    return time.perf_counter() - t, torch.cuda.max_memory_allocated() / 2 ** 30, r


def _stats(times):
    """Median and range of each leg's per-call seconds, and the ratio of the medians."""
    med = {k: statistics.median(v) for k, v in times.items()}
    return dict(dropin_s=med["dropin"], dropin_range_s=[min(times["dropin"]), max(times["dropin"])], reference_s=med["reference"],
                reference_range_s=[min(times["reference"]), max(times["reference"])], speedup=med["reference"] / med["dropin"])


def _card():
    try:
        q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True, text=True)
        return q.stdout.strip().splitlines()[0]
    except Exception:  # noqa: BLE001
        return torch.cuda.get_device_name()


def bench_filter(name, V, H, W, reps, card):
    import test_gpu_depth_filter as tg
    import test_depth_filter_oracle as tdo
    case = tg._big_case(V, H, W, seed=V)
    args = tg._inputs(case)
    opt = tdo._opt(case)
    legs = dict(dropin=lambda: depth_filter.filter_by_masks_gpu(*args, opt), reference=lambda: ref_filter(*args, opt))
    times = {k: [] for k in legs}
    peak, counts = {}, {}
    for k, fn in legs.items():                       # warm-up
        fn()
    for _ in range(reps):
        for k, fn in legs.items():
            t, m, out = _timed(fn)
            times[k].append(t)
            peak[k] = m
            counts[k] = [len(o[0]) if isinstance(o, tuple) else len(o) for o in (out if k == "reference" else out[0])]
    print(json.dumps(dict(case=name, views=V, H=H, W=W, pixel_pairs=V * (V - 1) * H * W,
                          reps=reps, **_stats(times), peak_gib=peak,
                          counts_agree=counts["dropin"] == counts["reference"], kept=dict(dropin=sum(counts["dropin"]),
                          reference=sum(counts["reference"])), views_whose_counts_differ=sum(a != b for a, b in zip(counts["dropin"],
                          counts["reference"])), card=card)), flush=True)


def bench_alpha(name, N, reps, card, V=100, H=800, W=800):
    import test_depth_filter_oracle as tdo
    case = tdo.alpha_case(N=8, V=V, H=H, W=W, seed=1)
    g = torch.Generator("cuda").manual_seed(0)
    pts = torch.empty((N, 3), device="cuda").uniform_(-1.2, 1.2, generator=g)
    pts[:, 2] += 3.0
    alpha = (torch.rand((V, H, W), device="cuda", generator=g) > 0.002).float()
    Ks = torch.from_numpy(case["K"]).cuda()
    w2c = torch.from_numpy(case["w2c"]).cuda()
    opt = types.SimpleNamespace(alpha_range=1, inall_img=1)
    nf = (0.5, 6.0)
    legs = dict(dropin=lambda: depth_filter.alpha_masking(pts, [a[None] for a in alpha], list(Ks), None, list(w2c), nf, opt=opt),
                reference=lambda: ref_alpha(pts, list(alpha), list(Ks), list(w2c), nf))
    times = {k: [] for k in legs}
    peak, kept = {}, {}
    for fn in legs.values():
        fn()
    for _ in range(reps):
        for k, fn in legs.items():
            t, m, out = _timed(fn)
            times[k].append(t)
            peak[k] = m
            kept[k] = int(out.sum())
    print(json.dumps(dict(case=name, points=N, views=V, H=H, W=W, reps=reps, **_stats(times), peak_gib=peak, counts_agree=kept["dropin"] == kept["reference"],
                          kept=kept, card=card)), flush=True)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=3)
    ap.add_argument("--only", default="dtu,n360,alpha10m,alpha50m")
    a = ap.parse_args()
    if not torch.cuda.is_available():
        sys.exit("bench_depth_filter.py needs a CUDA device")
    card = _card()
    only = a.only.split(",")
    if "dtu" in only:
        bench_filter("dtu", 49, 512, 640, a.reps, card)
    if "n360" in only:
        bench_filter("n360", 100, 800, 800, a.reps, card)
    if "alpha10m" in only:
        bench_alpha("alpha10m", 10_000_000, a.reps, card)
    if "alpha50m" in only:
        bench_alpha("alpha50m", 50_000_000, a.reps, card)


if __name__ == "__main__":
    main()
