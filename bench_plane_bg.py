"""The plane background of the DTU scripts (bgmodel plane): run/train_ft.py's create_all_bg loop (:549-575) -- gen_bg_points and
set_bg on every H*W ray of every frame -- with pointnerf_b200.plane_bg against the reference expression of
models/mvs/mvs_utils.py:299-421 and models/mvs_points_volumetric_model.py:272-310, restated here: the projections on the device, the
images on the host and grid_sample on the CPU (gen_points_filter_embeddings keeps them there, train_ft.py:87), the result copied back.

    python bench_plane_bg.py --frames 49 --ref-frames 4 --rounds 2

Workload: 49 frames of 512 x 640 rays (a DTU test set) from cameras on an arc, G in {16, 64} views (one per MVS view group) and
N in {1M, 4M} points on a seeded bumpy surface, a plane behind it.  Each round runs both legs, so they alternate within one process:
the reference expression on its first --ref-frames frames (every frame costs the same there: nothing is cached), then the drop-in on
all frames from a cleared cache (the first frame uploads the images and builds the masks).  Every timed window ends in a device
synchronisation.  Peak memory: torch.cuda.max_memory_allocated over the first frame of each leg, minus what was allocated before.
Also reported, over the frames both legs ran: the largest colour difference and the number of rays whose bg is zero in one leg only.
Prints one JSON line with the card name and power limit next to the numbers.  Writes nothing.
"""
import argparse
import json
import math
import statistics
import time
import types

import torch
import torch.nn.functional as Fn

from bench_voxelize import card
from pointnerf_b200 import plane_bg

H, W = 512, 640
PLANE_COLOR = (0.6, 0.4, 0.3)


def _rot(yaw, pitch):
    cy, sy, cp, sp = math.cos(yaw), math.sin(yaw), math.cos(pitch), math.sin(pitch)
    ry = torch.tensor([[cy, 0, sy], [0, 1, 0], [-sy, 0, cy]], dtype=torch.float64)
    rx = torch.tensor([[1, 0, 0], [0, cp, -sp], [0, sp, cp]], dtype=torch.float64)
    return ry @ rx


def _camera(yaw, pitch, centre):
    R = _rot(yaw, pitch)
    c = centre - R @ torch.tensor([0, 0, 3.0], dtype=torch.float64)
    return R, c


def scene_of(G, N, frames, dev, seed=0):
    g = torch.Generator().manual_seed(seed)
    f = 1.2 * W
    uv = torch.rand((N, 2), generator=g) - 0.5
    z = 3.0 + 0.3 * torch.sin(4 * uv[:, 0]) * torch.cos(3 * uv[:, 1])
    xyz = torch.stack([uv[:, 0] * W / f * z, uv[:, 1] * H / f * z, z], -1).float().to(dev)
    centre = torch.tensor([0, 0, 3.0], dtype=torch.float64)
    K = torch.tensor([[f, 0, W / 2], [0, f, H / 2], [0, 0, 1]], dtype=torch.float32)
    w2cs, Ks, imgs = [], [], []
    for k in range(G):
        R, c = _camera(-0.6 + 1.2 * k / max(G - 1, 1), 0.15 * (-1) ** k, centre)
        w = torch.eye(4, dtype=torch.float64)
        w[:3, :3] = R.T
        w[:3, 3] = -R.T @ c
        w2cs.append(w.float().to(dev)[None, None])
        Ks.append(K.to(dev)[None])
        pc = torch.tensor(PLANE_COLOR)[None, :, None, None]
        imgs.append((pc + (torch.rand((1, 3, H, W), generator=g) - 0.5) * 0.12).contiguous())   # on the host, as the scripts keep them
    px, py = torch.meshgrid(torch.arange(W, dtype=torch.float64), torch.arange(H, dtype=torch.float64), indexing="xy")
    d_cam = torch.stack([(px.reshape(-1) + 0.5 - W / 2) / f, (py.reshape(-1) + 0.5 - H / 2) / f, torch.ones(H * W, dtype=torch.float64)], -1)
    d_cam = d_cam / d_cam.norm(dim=-1, keepdim=True)
    batches = []
    n = torch.tensor([0.05, -0.4, 0.9])
    for i in range(frames):
        R, c = _camera(-0.5 + 1.0 * i / max(frames - 1, 1), 0.1, centre)
        batches.append(dict(campos=c.float().to(dev)[None], raydir=(d_cam @ R.T).float().to(dev)[None],
                            plane_pnt=torch.tensor([[0, 0, 3.6]]), plane_normal=(n / n.norm())[None],
                            plane_color=torch.tensor([PLANE_COLOR], device=dev)))
    return xyz, imgs, w2cs, Ks, [[H, W]] * G, batches


# ------------------------------------------------------------------------------------------------ the reference expression
def ref_gen_bg_points(batch):
    dev = batch["campos"].device
    p_co = torch.as_tensor(batch["plane_pnt"][0], dtype=torch.float32, device=dev)[None, None, :]
    p_no = torch.as_tensor(batch["plane_normal"][0], dtype=torch.float32, device=dev)[None, None, :]
    cam_pos, raydir = batch["campos"], batch["raydir"]
    dot = torch.sum(p_no * raydir, dim=-1)
    board_mask = dot >= 1e-3
    dot_valid = dot[board_mask][None, :]
    w = cam_pos[None, :, :] - p_co
    fac = -torch.sum(p_no * w, dim=-1) / dot_valid
    ray_dir_valid = raydir[:, board_mask[0], :] * fac[..., None]
    out = torch.zeros_like(raydir)
    out[:, board_mask[0], :] = cam_pos[None, ...] + ray_dir_valid
    return out


def _project(c2w, w2c, intrinsic, xyz, HD, WD):
    src_cam_xyz = torch.cat([xyz, torch.ones_like(xyz[:, :, 0:1])], dim=-1) @ c2w.transpose(1, 2) @ w2c.transpose(1, 2)
    src_grid = ((src_cam_xyz[..., :3] / src_cam_xyz[..., 2:3]) @ intrinsic.transpose(1, 2))[..., :2]
    mask = torch.prod(torch.cat([torch.ge(src_grid, torch.zeros([1, 1, 2], device=src_grid.device)),
                                 torch.le(src_grid, torch.tensor([[[WD - 1, HD - 1]]], device=src_grid.device))], dim=-1),
                      dim=-1, keepdim=True, dtype=torch.int8) > 0
    return src_grid, mask, torch.ceil(src_grid)


def ref_set_bg(xyz_sect, pts, img_lst, w2cs_lst, intrinsics_all, HDWD_lst, plane_color):
    c2w = torch.eye(4, device=xyz_sect.device, dtype=torch.float32)[None, ...]
    warped = []
    for imgs, w2c, intrinsics, (HD, WD) in zip(img_lst, w2cs_lst, intrinsics_all, HDWD_lst):
        w2c = w2c[:, 0, ...]
        src_grid, mask, hard = _project(c2w, w2c, intrinsics, xyz_sect, HD, WD)
        src_grid[..., 0] = src_grid[..., 0] / ((WD - 1.0) / 2.0) - 1.0
        src_grid[..., 1] = src_grid[..., 1] / ((HD - 1.0) / 2.0) - 1.0
        hard_valid = hard[:, mask[0, :, 0], :]
        _, fmask, fhard = _project(c2w, w2c, intrinsics, pts[None], HD, WD)
        fh = fhard[:, fmask[0, ..., 0], :].long()
        fg = torch.zeros([HD, WD], dtype=torch.int8, device=pts.device)
        fg[fh[0, ..., 1], fh[0, ..., 0]] = 1
        mask[0, mask[0, ..., 0].clone(), 0] = fg[hard_valid[0, ..., 1].long(), hard_valid[0, ..., 0].long()] < 1
        grid = src_grid[:, mask[0, ..., 0], :].cpu()
        s = Fn.grid_sample(imgs[0:1], grid[:, None, ...], mode="bilinear", padding_mode="zeros", align_corners=True)
        s = s.permute(0, 2, 3, 1).view(1, grid.shape[1], 3).to(xyz_sect.device)
        full = torch.zeros([1, mask.shape[1], 3], device=xyz_sect.device)
        full[0, mask[0, :, 0], :] = s
        warped.append(full)
    warped = torch.stack(warped, dim=-2)
    fit = torch.prod(torch.logical_and(warped >= (plane_color - 0.03), warped <= plane_color + 0.03), dim=-1)
    nofit = (1 - fit).nonzero()
    warped[0, nofit[..., 1], nofit[..., 2], :] = 0
    return torch.max(warped, dim=-2)[0]


# ------------------------------------------------------------------------------------------------ the two legs
def _timed(dev, fn):
    torch.cuda.synchronize(dev)
    t0 = time.perf_counter()
    out = fn()
    torch.cuda.synchronize(dev)
    return out, (time.perf_counter() - t0) * 1e3


def run_reference(dev, sc, frames):
    xyz, imgs, w2cs, Ks, hdwd, batches = sc
    outs, ms = [], []
    for b in batches[:frames]:
        o, t = _timed(dev, lambda: ref_set_bg(ref_gen_bg_points(b), xyz, imgs, w2cs, Ks, hdwd, b["plane_color"]))
        outs.append(o)
        ms.append(t)
    return outs, ms


def run_dropin(dev, sc, model):
    xyz, imgs, w2cs, Ks, hdwd, batches = sc
    plane_bg.reset(model)

    def frame(b):
        return plane_bg.set_bg(model, plane_bg.gen_bg_points(b), imgs, [None] * len(imgs), w2cs, Ks, hdwd, b["plane_color"])[0]

    first, t_first = _timed(dev, lambda: frame(batches[0]))
    rest, t_rest = _timed(dev, lambda: [frame(b) for b in batches[1:]])
    return [first] + rest, t_first, t_rest / max(len(batches) - 1, 1)


def bench_case(args, dev, G, N):
    sc = scene_of(G, N, args.frames, dev)
    model = types.SimpleNamespace(neural_points=types.SimpleNamespace(xyz=sc[0]))
    peak = {}
    for leg in ("reference_expr", "dropin"):
        torch.cuda.empty_cache()
        torch.cuda.synchronize(dev)
        base = torch.cuda.memory_allocated(dev)
        torch.cuda.reset_peak_memory_stats(dev)
        if leg == "dropin":
            plane_bg.reset(model)
            plane_bg.set_bg(model, plane_bg.gen_bg_points(sc[5][0]), sc[1], [None] * G, sc[2], sc[3], sc[4], sc[5][0]["plane_color"])
        else:
            ref_set_bg(ref_gen_bg_points(sc[5][0]), sc[0], sc[1], sc[2], sc[3], sc[4], sc[5][0]["plane_color"])
        torch.cuda.synchronize(dev)
        peak[leg] = (torch.cuda.max_memory_allocated(dev) - base) / 2 ** 20
        plane_bg.reset(model)
    ref_first, ref_rest, drop_first, drop_rest = [], [], [], []
    max_d, zero_flip, compared = 0.0, 0, 0
    for _ in range(args.rounds):
        r_out, r_ms = run_reference(dev, sc, args.ref_frames)
        d_out, d_first, d_rest = run_dropin(dev, sc, model)
        ref_first.append(r_ms[0])
        ref_rest += r_ms[1:]
        drop_first.append(d_first)
        drop_rest.append(d_rest)
        for a, b in zip(r_out, d_out):
            max_d = max(max_d, float((a - b).abs().max()))
            zero_flip += int(((a == 0).all(-1) != (b == 0).all(-1)).sum())
            compared += int(a.shape[1])
        del r_out, d_out
    ref_steady = statistics.median(ref_rest) if ref_rest else None
    steady = statistics.median(drop_rest)
    total_ref = ref_steady * args.frames if ref_steady is not None else None
    total_drop = statistics.median(drop_first) + steady * (args.frames - 1)
    del sc, model
    torch.cuda.empty_cache()
    return dict(views=G, points=N, frames=args.frames, rays_per_frame=H * W,
                reference_expr=dict(first_frame_ms=round(statistics.median(ref_first), 1),
                                    steady_frame_ms=round(ref_steady, 1) if ref_steady is not None else None,
                                    frames_timed=args.ref_frames, peak_mb_first_frame=round(peak["reference_expr"], 1),
                                    loop_s_estimated=round(total_ref / 1e3, 2) if total_ref is not None else None),
                dropin=dict(first_frame_ms=round(statistics.median(drop_first), 2), steady_frame_ms=round(steady, 3),
                            peak_mb_first_frame=round(peak["dropin"], 1), loop_s=round(total_drop / 1e3, 3)),
                rays_compared=compared, max_abs_color_diff=max_d, rays_zero_in_one_leg_only=zero_flip)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--frames", type=int, default=49)
    ap.add_argument("--ref-frames", type=int, default=4)
    ap.add_argument("--rounds", type=int, default=2)
    ap.add_argument("--views", type=int, nargs="+", default=[16, 64])
    ap.add_argument("--points", type=int, nargs="+", default=[1_000_000, 4_000_000])
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise RuntimeError("bench_plane_bg.py needs a CUDA device: the product has no CPU path")
    args.ref_frames = max(1, min(args.ref_frames, args.frames))
    dev = torch.device("cuda", 0)
    res = [bench_case(args, dev, G, N) for G in args.views for N in args.points]
    name, smi = card()
    print(json.dumps(dict(metric="create_all_bg-shaped loop (gen_bg_points + set_bg per 512x640 frame): pointnerf_b200.plane_bg vs "
                                 "the reference expression (CPU grid_sample on host images)", gpu=name, nvidia_smi_name_power_limit=smi,
                          rounds=args.rounds, torch_threads=torch.get_num_threads(), cases=res)))


if __name__ == "__main__":
    main()
