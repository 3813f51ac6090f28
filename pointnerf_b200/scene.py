"""Seeded synthetic scenes + camera rays for the hot-path configs of BASELINE.json (SURVEY.md 8d).

There is no dataset / checkpoint offline, so every test and bench line runs on this generator:
a thin noisy spherical shell of neural points (two crossings per hitting ray), a pinhole camera
as in the reference's NeRF-Synthetic dataset class
(/root/reference/data/nerf_synth360_ft_dataset.py:381, :557-646) and rays from
get_dtu_raydir (/root/reference/data/data_utils.py:55-69; +0.5 px, un-normalised, z_cam = 1).
"""
import math
from dataclasses import dataclass, field

import numpy as np
import torch


@dataclass
class SceneConfig:
    name: str
    N: int
    R_s: float
    vsize: float
    vscale: int = 2
    kernel_size: int = 3
    query_size: int = 3
    radius_limit_scale: float = 4.0
    SR: int = 24
    K: int = 8
    P: int = 16
    D: int = 400
    H: int = 800
    W: int = 800
    near: float = 2.0
    far: float = 6.0
    campos: tuple = (0.0, 0.0, -4.0)
    seed: int = 1234
    shape: str = "shell"           # "shell" | "box"
    box: tuple = (8.0, 6.0, 3.0)   # for shape == "box" (config 5)
    fov_x: float = 0.6911112       # nerf_synth360_ft_dataset.py:381


CONFIGS = {
    # BASELINE.json configs[0..4]; sizes per SURVEY 8(d)
    "chair_plumbing": SceneConfig("chair_plumbing", N=10_000, R_s=0.6, vsize=0.02, P=32),
    "lego_render": SceneConfig("lego_render", N=400_000, R_s=1.0, vsize=0.004, P=16),
    "ship_optimise": SceneConfig("ship_optimise", N=600_000, R_s=1.0, vsize=0.004, P=16),
    "truck_8gpu": SceneConfig("truck_8gpu", N=2_000_000, R_s=0.8, vsize=0.002, kernel_size=5, P=16,
                              H=540, W=960, near=0.0, far=3.5, campos=(0.0, 0.0, -2.2)),
    "scannet_8gpu": SceneConfig("scannet_8gpu", N=5_000_000, R_s=0.0, vsize=0.008, P=30, H=480, W=640,
                                near=0.1, far=8.0, campos=(0.5, 0.3, 0.2), shape="box"),
    # small cases for parity tests
    "tiny": SceneConfig("tiny", N=3_000, R_s=0.6, vsize=0.03, P=32, H=64, W=64),
}


def make_points(cfg: SceneConfig, device="cpu", emb_dim=32):
    """xyz[N,3], embedding[1,N,emb_dim], color[1,N,3], dir[1,N,3], conf[1,N,1], Rw2c[3,3] (fp32).  emb_dim 32 (the default) gives
    the seeded values of every existing fixture; the DTU configuration (point_features_dim 63, point_*_mode "01") takes 56 image
    features and prepends colour, dir and conf itself (NeuralPoints.set_points)."""
    g = torch.Generator().manual_seed(cfg.seed)
    N = cfg.N
    if cfg.shape == "shell":
        d = torch.randn(N, 3, generator=g)
        d = d / d.norm(dim=-1, keepdim=True)
        r = cfg.R_s + cfg.vsize * torch.randn(N, 1, generator=g)
        xyz = r * d
        pdir = d
    else:  # inside walls of a box, uniform per area, normal noise
        bx, by, bz = cfg.box
        areas = torch.tensor([by * bz, by * bz, bx * bz, bx * bz, bx * by, bx * by])
        face = torch.multinomial(areas / areas.sum(), N, replacement=True, generator=g)
        u = torch.rand(N, 2, generator=g) - 0.5
        nrm = cfg.vsize * torch.randn(N, generator=g)
        xyz = torch.zeros(N, 3)
        pdir = torch.zeros(N, 3)
        half = torch.tensor([bx, by, bz]) / 2
        for f in range(6):
            m = face == f
            ax = f // 2
            sgn = 1.0 if f % 2 == 0 else -1.0
            oth = [a for a in range(3) if a != ax]
            xyz[m, ax] = sgn * half[ax] + nrm[m]
            xyz[m, oth[0]] = u[m, 0] * 2 * half[oth[0]]
            xyz[m, oth[1]] = u[m, 1] * 2 * half[oth[1]]
            pdir[m, ax] = -sgn
    emb = 0.5 * torch.randn(1, N, emb_dim, generator=g)
    color = torch.rand(1, N, 3, generator=g)
    conf = 0.1 + 0.9 * torch.rand(1, N, 1, generator=g)
    out = dict(xyz=xyz.float().contiguous(), embedding=emb, color=color, dir=pdir[None].float().contiguous(),
               conf=conf, Rw2c=torch.eye(3))
    return {k: v.to(device) for k, v in out.items()}


def edit_frames(xyz, seed=11):
    """Per-point Rw2c [N,3,3] shaped like a scene edit (the reference's run/editing.py:186-212 stores the rotation of each object's
    rigid transform on its points): the cloud split by sign(x) into two objects, rotated by seeded angles in [0.4, 1.2) rad about z
    (x < 0) and about x (x >= 0).  Samples near the seam x = 0 have neighbours in both frames."""
    g = torch.Generator().manual_seed(seed)
    a, b = (0.4 + 0.8 * torch.rand(2, generator=g)).tolist()
    ca, sa, cb, sb = math.cos(a), math.sin(a), math.cos(b), math.sin(b)
    Rz = torch.tensor([[ca, -sa, 0.0], [sa, ca, 0.0], [0.0, 0.0, 1.0]], dtype=torch.float32)
    Rx = torch.tensor([[1.0, 0.0, 0.0], [0.0, cb, -sb], [0.0, sb, cb]], dtype=torch.float32)
    left = (xyz[:, 0] < 0)[:, None, None]
    return torch.where(left, Rz.to(xyz.device), Rx.to(xyz.device)).contiguous()


def make_intrinsic(cfg: SceneConfig):
    f = 0.5 * cfg.W / math.tan(0.5 * cfg.fov_x)
    return np.array([[f, 0, cfg.W / 2], [0, f, cfg.H / 2], [0, 0, 1]], dtype=np.float32)


def make_rays(cfg: SceneConfig, pixels=None):
    """pixels: None = full image in row-major (y outer, x inner) order, or an [R,2] array of (px,py).
    Returns dict with raydir[1,R,3] f32 (un-normalised), pixel_idx[1,R,2] f32, campos[1,3],
    camrotc2w[1,3,3], intrinsic[1,3,3], near[1,1], far[1,1], h[1], w[1]."""
    K = make_intrinsic(cfg)
    if pixels is None:
        px, py = np.meshgrid(np.arange(cfg.W).astype(np.float32), np.arange(cfg.H).astype(np.float32))
        pix = np.stack((px, py), axis=-1).reshape(-1, 2)
    else:
        pix = np.asarray(pixels, np.float32).reshape(-1, 2)
    x = (pix[:, 0] + 0.5 - K[0, 2]) / K[0, 0]
    y = (pix[:, 1] + 0.5 - K[1, 2]) / K[1, 1]
    dirs = np.stack([x, y, np.ones_like(x)], axis=-1) @ np.eye(3, dtype=np.float32).T
    return dict(
        raydir=torch.from_numpy(dirs.astype(np.float32))[None],
        pixel_idx=torch.from_numpy(pix)[None],
        campos=torch.tensor([cfg.campos], dtype=torch.float32),
        camrotc2w=torch.eye(3)[None],
        intrinsic=torch.from_numpy(K)[None],
        near=torch.tensor([[cfg.near]], dtype=torch.float32),
        far=torch.tensor([[cfg.far]], dtype=torch.float32),
        h=torch.tensor([cfg.H]), w=torch.tensor([cfg.W]),
        bg_color=torch.ones(1, 3),
    )


def centre_patch(cfg: SceneConfig, side):
    x0, y0 = cfg.W // 2 - side // 2, cfg.H // 2 - side // 2
    px, py = np.meshgrid(np.arange(x0, x0 + side), np.arange(y0, y0 + side))
    return np.stack((px, py), -1).reshape(-1, 2).astype(np.float32)


def ranges_for(cfg: SceneConfig):
    if cfg.shape == "shell":
        e = cfg.R_s + 0.1
        return (-e, -e, -e, e, e, e)
    return (-10.0,) * 3 + (10.0,) * 3
