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


def orbit_rotation(yaw=0.7, pitch=0.3):
    """camrotc2w [3,3] (fp32) of a camera orbited about the origin: yaw about the world y axis after pitch about x.  The shell configs'
    cameras look at the origin along +z, so R @ cfg.campos looks at it along R[:, 2] and the shell stays between near and far."""
    cy, sy, cp, sp = math.cos(yaw), math.sin(yaw), math.cos(pitch), math.sin(pitch)
    Ry = np.array([[cy, 0.0, sy], [0.0, 1.0, 0.0], [-sy, 0.0, cy]])
    Rx = np.array([[1.0, 0.0, 0.0], [0.0, cp, -sp], [0.0, sp, cp]])
    return (Ry @ Rx).astype(np.float32)


def make_rays(cfg: SceneConfig, pixels=None, camrotc2w=None, bg_color=(1.0, 1.0, 1.0)):
    """pixels: None = full image in row-major (y outer, x inner) order, or an [R,2] array of (px,py).
    camrotc2w: None (the identity camera of every config) or a [3,3] rotation (e.g. orbit_rotation()) that orbits the camera about the
    origin: campos = R @ cfg.campos, raydir = R @ d_cam.  bg_color: the three channels of the background (white by default).
    Returns dict with raydir[1,R,3] f32 (un-normalised), pixel_idx[1,R,2] f32, campos[1,3],
    camrotc2w[1,3,3], intrinsic[1,3,3], near[1,1], far[1,1], h[1], w[1], bg_color[1,3]."""
    K = make_intrinsic(cfg)
    if pixels is None:
        px, py = np.meshgrid(np.arange(cfg.W).astype(np.float32), np.arange(cfg.H).astype(np.float32))
        pix = np.stack((px, py), axis=-1).reshape(-1, 2)
    else:
        pix = np.asarray(pixels, np.float32).reshape(-1, 2)
    x = (pix[:, 0] + 0.5 - K[0, 2]) / K[0, 0]
    y = (pix[:, 1] + 0.5 - K[1, 2]) / K[1, 1]
    rot = np.eye(3, dtype=np.float32) if camrotc2w is None else np.asarray(camrotc2w, np.float32).reshape(3, 3)
    dirs = np.stack([x, y, np.ones_like(x)], axis=-1) @ rot.T
    campos = cfg.campos if camrotc2w is None else tuple((rot @ np.asarray(cfg.campos, np.float32)).tolist())
    return dict(
        raydir=torch.from_numpy(dirs.astype(np.float32))[None],
        pixel_idx=torch.from_numpy(pix)[None],
        campos=torch.tensor([campos], dtype=torch.float32),
        camrotc2w=torch.from_numpy(rot.copy())[None],
        intrinsic=torch.from_numpy(K)[None],
        near=torch.tensor([[cfg.near]], dtype=torch.float32),
        far=torch.tensor([[cfg.far]], dtype=torch.float32),
        h=torch.tensor([cfg.H]), w=torch.tensor([cfg.W]),
        bg_color=torch.tensor([list(bg_color)], dtype=torch.float32),
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


# ---- DTU-like scenes of the perspective-frustum query (wcoord_query 0, NN 2; the DTU scripts' query options) ----
@dataclass
class FrustumConfig:
    name: str
    N: int = 30_000
    H: int = 120
    W: int = 160
    focal: float = 200.0
    near: float = 2.0
    far: float = 4.725
    z_depth_dim: int = 400
    vscale: tuple = (2, 2, 1)
    kernel_size: tuple = (3, 3, 3)
    query_size: tuple = (3, 3, 3)
    SR: int = 40
    K: int = 8
    P: int = 20
    radius_limit_scale: float = 0.0
    depth_limit_scale: float = 0.0
    seed: int = 4321


FRUSTUM_CONFIGS = {
    "dtu_surface": FrustumConfig("dtu_surface"),
    # non-zero limits: the radius / depth branch of the layered search
    "dtu_surface_limits": FrustumConfig("dtu_surface_limits", radius_limit_scale=1.5, depth_limit_scale=1.2),
}


def make_frustum_scene(cfg: FrustumConfig):
    """A bumpy surface about 2.5 units in front of a pinhole camera, plus 2 % of points scattered around the frustum (some of them
    within one voxel outside the grid, where truncation and floor differ).  Returns numpy xyz_cam [N,3], pers [N,3] (x/z, y/z, z as
    NeuralPoints.w2pers forms it), the world frame (camrotc2w [3,3], campos [3], xyz_w [N,3]), intrinsic [3,3] and the full-frame
    pixel_idx [H*W,2] (x, y; y outer)."""
    g = np.random.RandomState(cfg.seed)
    n_out = cfg.N // 50
    n_surf = cfg.N - n_out
    u = g.uniform(-0.45, 0.45, n_surf) * cfg.W / cfg.focal
    v = g.uniform(-0.45, 0.45, n_surf) * cfg.H / cfg.focal
    z = 2.5 + 0.25 * np.sin(3.0 * u) * np.cos(2.0 * v) + 0.6 * (u * u + v * v) + 0.004 * g.randn(n_surf)
    surf = np.stack([u * z, v * z, z], -1)
    xr, yr = 0.5 * cfg.W / cfg.focal + 0.01, 0.5 * cfg.H / cfg.focal + 0.01
    zo = g.uniform(cfg.near - 0.02, cfg.far + 0.02, n_out)
    out = np.stack([g.uniform(-xr, xr, n_out) * zo, g.uniform(-yr, yr, n_out) * zo, zo], -1)
    xyz_cam = np.concatenate([surf, out])[g.permutation(cfg.N)].astype(np.float32)
    pers = np.stack([xyz_cam[:, 0] / xyz_cam[:, 2], xyz_cam[:, 1] / xyz_cam[:, 2], xyz_cam[:, 2]], -1).astype(np.float32)
    a = 0.3
    camrotc2w = np.array([[math.cos(a), 0.0, math.sin(a)], [0.0, 1.0, 0.0], [-math.sin(a), 0.0, math.cos(a)]], np.float32)
    campos = np.array([0.2, -0.1, -0.3], np.float32)
    xyz_w = (xyz_cam @ camrotc2w.T + campos).astype(np.float32)
    intrinsic = np.array([[cfg.focal, 0, cfg.W / 2], [0, cfg.focal, cfg.H / 2], [0, 0, 1]], np.float32)
    px, py = np.meshgrid(np.arange(cfg.W), np.arange(cfg.H))
    pixel_idx = np.stack((px, py), -1).reshape(-1, 2).astype(np.int32)
    return dict(xyz_cam=xyz_cam, pers=pers, camrotc2w=camrotc2w, campos=campos, xyz_w=xyz_w, intrinsic=intrinsic, pixel_idx=pixel_idx)


def frustum_opt(cfg: FrustumConfig, is_train=False, **over):
    """The querier options of the DTU scripts (dev_scripts/dtu_test_inf/inftest_scan*.sh) for one FrustumConfig."""
    from types import SimpleNamespace
    o = SimpleNamespace(inverse=0, NN=2, K=cfg.K, SR=cfg.SR, P=cfg.P, max_o=None, z_depth_dim=cfg.z_depth_dim, vscale=list(cfg.vscale),
                        kernel_size=list(cfg.kernel_size), query_size=list(cfg.query_size), radius_limit_scale=cfg.radius_limit_scale,
                        depth_limit_scale=cfg.depth_limit_scale, gpu_maxthr=1024, is_train=is_train, shpnt_jitter="uniform",
                        wcoord_query=0)
    for k, v in over.items():
        setattr(o, k, v)
    return o


def make_frustum_points(cfg: FrustumConfig, s, emb_dim=63):
    """Seeded neural-point attributes for a frustum scene (world xyz from make_frustum_scene): the dict the shading oracles take."""
    g = torch.Generator().manual_seed(cfg.seed + 1)
    N = s["xyz_w"].shape[0]
    d = torch.randn(N, 3, generator=g)
    return dict(xyz=torch.from_numpy(s["xyz_w"]), embedding=0.5 * torch.randn(1, N, emb_dim, generator=g),
                color=torch.rand(1, N, 3, generator=g), dir=(d / d.norm(dim=-1, keepdim=True))[None],
                conf=0.1 + 0.9 * torch.rand(1, N, 1, generator=g), Rw2c=torch.eye(3))
