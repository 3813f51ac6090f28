"""TEST INFRASTRUCTURE ONLY (imported by tests/test_oracle_frustum_fused.py and tests/test_gpu_frustum_fused.py; not a test module).

The reference's eager shading of a perspective-frustum query result, as oracle/shade_oracle_frustum.py restates it, with what the
fused-module checks need beyond that restatement:
  agg_intrp_order  2 (alpha per neighbour, then the weighted sum) or 1 (alpha_branch on the K-aggregated feature,
                   point_aggregators.py:573-587), as oracle/shade_oracle.py takes it
  slopes           None (LeakyReLU) or the per-unit slopes of the 7 LeakyReLU layers (another computation's masks), as
                   oracle/shade_oracle.py takes them
  decoded          (sigma, rgb) of every sample [R',SR,4] in the result, for the per-sample comparison of DESIGN.md §6 item 6, with
                   h-bar, weight and conf_coefficient
  march            the ray distances and ray_march alone, on a given (sigma, rgb): the compositing kernel's check on the shading
                   kernels' own output
  scenes           point sets for tests/test_gpu_frustum_f64.py in the camera of scene.make_frustum_scene (frustum_scene), the CPU
                   query oracle on them (oracle_query), and the backward's LeakyReLU masks of a frustum training step (kernel_slopes)
tests/test_oracle_frustum_fused.py holds it bit for bit to oracle/shade_oracle_frustum.shade (order 2, no slopes) on the frustum
query's tuple and to oracle/shade_oracle.shade (orders 1 and 2, with and without slopes) on the world query's inputs.
"""
import contextlib
import functools

import numpy as np
import torch
import torch.nn.functional as F

from oracle.shade_oracle import _act, _lin, positional_encoding, w2pers


def shade(points, mlp, sample_pidx, sample_loc, sample_loc_w, sample_ray_dirs, campos, camrotc2w, vsize, bg_color, dtype=torch.float64,
          agg_intrp_order=2, slopes=None):
    """Arguments as oracle/shade_oracle_frustum.shade (the querier's tuple without the batch dimension; vsize: the querier's).
    Returns march()'s dict (ray_color [R',3], opacity [R',SR], bg_T [R',1], ray_dist, blend_weight) with decoded [R',SR,4],
    ray_valid [R',SR], weight and conf_coefficient [R',SR,K] (the reference's output keys) and hbar [R'*SR,256]."""
    assert agg_intrp_order in (1, 2)
    cv = lambda t: t.to(dtype)  # noqa: E731
    xyz = cv(points["xyz"]); emb = cv(points["embedding"][0]); col = cv(points["color"][0])
    pdir = cv(points["dir"][0]); conf = cv(points["conf"][0]); Rw2c = cv(points["Rw2c"])
    mlp = {k: cv(v) for k, v in mlp.items()}
    sample_loc, sample_loc_w, sample_ray_dirs = cv(sample_loc), cv(sample_loc_w), cv(sample_ray_dirs)
    campos = cv(campos).reshape(3); camrotc2w = cv(camrotc2w).reshape(3, 3); bg_color = cv(bg_color).reshape(3)
    Rn, SR, K = sample_pidx.shape
    act = lambda x, layer: _act(x, slopes, layer)  # noqa: E731

    # gather (neural_points.py:706-717)
    pnt_mask = sample_pidx >= 0
    idx = torch.clamp(sample_pidx, min=0).reshape(-1).long()
    xyz_pers_all = w2pers(xyz, camrotc2w, campos)
    s_xyz = xyz[idx].view(Rn, SR, K, 3)
    s_xyz_pers = xyz_pers_all[idx].view(Rn, SR, K, 3)
    s_emb = emb[idx].view(Rn, SR, K, -1)
    s_col = col[idx].view(Rn, SR, K, 3)
    s_dir = pdir[idx].view(Rn, SR, K, 3)
    s_conf = conf[idx].view(Rn, SR, K, 1)

    # PointAggregator.forward (point_aggregators.py:727-814), agg_dist_pers 20, viewmlp (:488-644); the querier's own sample_loc and
    # per-sample sample_ray_dirs (:773-781)
    ray_valid = torch.any(pnt_mask, dim=-1)
    xdist = s_xyz_pers[..., 0] * s_xyz_pers[..., 2] - sample_loc[:, :, None, 0] * sample_loc[:, :, None, 2]
    ydist = s_xyz_pers[..., 1] * s_xyz_pers[..., 2] - sample_loc[:, :, None, 1] * sample_loc[:, :, None, 2]
    zdist = s_xyz_pers[..., 2] - sample_loc[:, :, None, 2]
    dists = torch.cat([s_xyz - sample_loc_w[..., None, :], torch.stack([xdist, ydist, zdist], dim=-1)], dim=-1)
    weight = pnt_mask * (1.0 / torch.clamp(torch.norm(dists[..., :3], dim=-1), min=1e-6))
    weight = weight / torch.clamp(torch.sum(weight, dim=-1, keepdim=True), min=1e-8)
    c0 = s_conf[..., 0]
    cc = c0 - (c0 - torch.clamp(c0, min=0.0001, max=1)).detach()
    wc = weight * cc
    Rt = Rw2c.transpose(-1, -2)
    viewdirs = sample_ray_dirs.reshape(-1, 3) @ Rt
    pe_view = positional_encoding(viewdirs, 4, ori=True)
    ori_viewdirs, pe_view = pe_view[..., :3], pe_view[..., 3:]
    sv = ray_valid.reshape(-1)
    pm = pnt_mask.reshape(-1)
    d_flat = dists.reshape(-1, 6)[pm]
    d_flat = torch.cat([d_flat[:, :3] @ Rt, d_flat[:, 3:]], dim=-1)
    f = s_emb.reshape(-1, s_emb.shape[-1])[pm]
    feat = torch.cat([f, positional_encoding(f, 3), positional_encoding(d_flat, 5)], dim=-1)
    feat = act(_lin(act(_lin(feat, mlp, "block1.0"), 0), mlp, "block1.2"), 1)
    dir_flat = s_dir.reshape(-1, 3)[pm] @ Rt
    ov = ori_viewdirs[:, None, :].expand(-1, K, -1).reshape(-1, 3)[pm]
    feat = torch.cat([feat, s_col.reshape(-1, 3)[pm], dir_flat - ov, torch.sum(dir_flat * ov, dim=-1, keepdim=True)], dim=-1)
    feat = act(_lin(act(_lin(feat, mlp, "block3.0"), 2), mlp, "block3.2"), 3)
    alpha = F.softplus(_lin(feat, mlp, "alpha_branch.0") - 1)
    pm_idx = pm.nonzero()[:, 0]
    alpha_h = torch.zeros(Rn * SR * K, 1, dtype=dtype).index_put((pm_idx,), alpha)
    feat_h = torch.zeros(Rn * SR * K, feat.shape[-1], dtype=dtype).index_put((pm_idx,), feat)
    wflat = wc.reshape(Rn * SR, K, 1)
    hbar = torch.sum(feat_h.view(Rn * SR, K, -1) * wflat, dim=-2)
    if agg_intrp_order == 2:
        sigma = torch.sum(alpha_h.view(Rn * SR, K, 1) * wflat, dim=-2)
    else:
        sigma = F.softplus(_lin(hbar, mlp, "alpha_branch.0") - 1)
    x = act(_lin(torch.cat([hbar, pe_view], dim=-1), mlp, "color_branch.0"), 4)
    x = act(_lin(act(_lin(x, mlp, "color_branch.2"), 5), mlp, "color_branch.4"), 6)
    rgb = torch.sigmoid(_lin(x, mlp, "color_branch.6")) * (1 + 2 * 0.001) - 0.001
    decoded = torch.cat([sigma, rgb], dim=-1)
    decoded = torch.where(sv[:, None], decoded, torch.zeros_like(decoded)).view(Rn, SR, 4)

    r = march(decoded, ray_valid, sample_loc, vsize, bg_color, dtype)
    return dict(r, decoded=decoded, ray_valid=ray_valid, weight=weight, conf_coefficient=cc, hbar=hbar)


def march(decoded, ray_valid, sample_loc, vsize, bg_color, dtype=torch.float64):
    """The ray distances of the frustum query and ray_march on a given decoded [R',SR,4] (sigma, rgb): the cumulative maximum of the
    querier's sample_loc[..., 2] (empty slots at near - vsize_z/2, jitter included), steps below 1e-8 or above 2 vsize_z replaced by
    vsize_z, the last slot vsize_z (neural_points_volumetric_model.py:271-279, diff_ray_marching.py:508-554).  shade() ends with it, so
    it is shade()'s arithmetic; the depth steps of fp32 sample_loc are exact in fp32 (consecutive depths within a factor 2), so float64
    takes the same replacement decisions as the kernels.  Returns dict(ray_dist, opacity, bg_T, blend_weight [R',SR,1], ray_color)."""
    decoded, sample_loc, bg_color = decoded.to(dtype), sample_loc.to(dtype), bg_color.to(dtype).reshape(3)
    Rn = decoded.shape[0]
    ray_dist = ray_dists(sample_loc, ray_valid, float(vsize[2]), dtype)
    opacity = 1 - torch.exp(-decoded[..., 0] * ray_valid.to(dtype) * ray_dist)
    acc = torch.cumprod(1. - opacity + 1e-10, dim=-1)
    bg_T = acc[:, -1:]
    acc_T = torch.cat([torch.ones(Rn, 1, dtype=dtype), acc[:, :-1]], dim=-1)
    blend_weight = opacity * acc_T
    ray_color = torch.sum(decoded[..., 1:4] * blend_weight[..., None], dim=-2) + bg_color.view(1, 3) * bg_T
    return dict(ray_dist=ray_dist, opacity=opacity, bg_T=bg_T, blend_weight=blend_weight[..., None], ray_color=ray_color)


def ray_dists(sample_loc, ray_valid, vz, dtype):
    """[R',SR] ray distances of march() (neural_points_volumetric_model.py:271-279)."""
    Rn = sample_loc.shape[0]
    z = torch.cummax(sample_loc[..., 2], dim=-1)[0]
    ray_dist = torch.cat([z[..., 1:] - z[..., :-1], torch.full((Rn, 1), vz, dtype=dtype)], dim=-1)
    m = torch.logical_or(ray_dist < 1e-8, ray_dist > 2 * vz).to(dtype)
    return (ray_dist * (1.0 - m) + m * vz) * ray_valid.to(dtype)


# ------------------------------------------------------------------------------------------------ scenes of the float64 checks
SCENES = ("dtu_surface", "dtu_surface_limits", "layers", "fog")


def _layers(g, cfg, n):
    """Three bumpy surfaces at depths 2.35, 2.75 and 3.3 (the depth voxel is 0.0068 long: tens of empty voxels between them), n points
    each over the whole frame."""
    out = []
    for i, z0 in enumerate((2.35, 2.75, 3.3)):
        u = g.uniform(-0.45, 0.45, n) * cfg.W / cfg.focal
        v = g.uniform(-0.45, 0.45, n) * cfg.H / cfg.focal
        z = z0 + 0.06 * np.sin(3.0 * u + i) * np.cos(2.0 * v) + 0.004 * g.randn(n)
        out.append(np.stack([u * z, v * z, z], -1))
    return np.concatenate(out)


# the fog slab of "fog": camera-frame x/z, y/z and depth ranges (pixels 60..90 x 44..74 of the 160 x 120 frame)
FOG_BOX = ((-0.1, 0.05), (-0.08, 0.07), (2.2, 3.25))


@functools.lru_cache(None)
def frustum_scene(name):
    """(cfg, s, points) of one scene: cfg a scene.FrustumConfig (query options), s as scene.make_frustum_scene returns it (the same
    rotated camera, 160 x 120 frame and intrinsic for every scene), points as scene.make_frustum_points.
      dtu_surface, dtu_surface_limits  scene.FRUSTUM_CONFIGS' own
      layers                           _layers: 3 x 8,000 points
      fog                              _layers with 4,000 points each, and 24,000 points uniform in FOG_BOX: its columns hold more
                                       than 128 dilated voxels"""
    from pointnerf_b200 import scene
    if name in scene.FRUSTUM_CONFIGS:
        cfg = scene.FRUSTUM_CONFIGS[name]
        s = scene.make_frustum_scene(cfg)
        return cfg, s, scene.make_frustum_points(cfg, s)
    cfg = scene.FRUSTUM_CONFIGS["dtu_surface"]
    s = scene.make_frustum_scene(cfg)
    g = np.random.RandomState(77)
    if name == "layers":
        xyz = _layers(g, cfg, 8000)
    elif name == "fog":
        n = 24000
        (u0, u1), (v0, v1), (z0, z1) = FOG_BOX
        u, v, z = g.uniform(u0, u1, n), g.uniform(v0, v1, n), g.uniform(z0, z1, n)
        xyz = np.concatenate([_layers(g, cfg, 4000), np.stack([u * z, v * z, z], -1)])
    else:
        raise KeyError(name)
    xyz_cam = xyz[g.permutation(len(xyz))].astype(np.float32)
    pers = np.stack([xyz_cam[:, 0] / xyz_cam[:, 2], xyz_cam[:, 1] / xyz_cam[:, 2], xyz_cam[:, 2]], -1).astype(np.float32)
    xyz_w = (xyz_cam @ s["camrotc2w"].T + s["campos"]).astype(np.float32)
    s = dict(s, xyz_cam=xyz_cam, pers=pers, xyz_w=xyz_w)
    return cfg, s, scene.make_frustum_points(cfg, s)


def fog_pixels(step=4):
    """Pixels (x, y) of the fog slab's columns, every step-th in x and y."""
    px, py = np.meshgrid(np.arange(61, 90, step), np.arange(45, 74, step))
    return np.stack((px, py), -1).reshape(-1, 2).astype(np.int32)


def oracle_query(name, pixels, **over):
    """The CPU frustum oracle (oracle/frustum_oracle.c) on a scene, query options of scene.frustum_opt with `over`.  Returns
    (opt, vsize, out) with out as frustum_oracle.query returns it."""
    from oracle import frustum_oracle
    from pointnerf_b200 import scene
    from pointnerf_b200 import query_point_indices as qpi
    cfg, s, _ = frustum_scene(name)
    opt = scene.frustum_opt(cfg, **over)
    rl, dl, ranges, vsize, vdim, svs, sdim, vscale = qpi.hyperparameters(opt, np.int64(cfg.H), np.int64(cfg.W), s["intrinsic"],
                                                                         np.float32(cfg.near), np.float32(cfg.far))
    out = frustum_oracle.query(s["pers"], ranges[:3], svs, sdim, vscale, opt.kernel_size, opt.query_size, opt.SR, opt.K, opt.P,
                               pixels, np.float32(rl ** 2), np.float32(dl ** 2), max_o=opt.max_o)
    return opt, vsize, out


def reach(out, vsize):
    """What a query result reaches: hit rays, capped columns, rays without any neighbour, valid samples that take the > 2 vsize_z
    replacement, the K-fill histogram of the valid samples (index = filled K slots)."""
    pidx = out["sample_pidx"]
    valid = (pidx >= 0).any(-1)
    z = np.maximum.accumulate(out["sample_loc"][..., 2], axis=-1)
    rd = z[:, 1:] - z[:, :-1]
    return dict(R2=int(pidx.shape[0]), capped=int(out["counters"]["n_col_capped"]), no_nb=int((~valid.any(-1)).sum()),
                gap=int(((rd > 2 * float(vsize[2])) & valid[:, :-1]).sum()),
                kfill=np.bincount((pidx >= 0).sum(-1)[valid], minlength=pidx.shape[2] + 1).tolist())


def kernel_slopes(net, q):
    """The LeakyReLU masks the backward of the last training step of a frustum module took (its recompute buffers,
    pnb_backward_tables) as `slopes=` of shade(): pair rows in the flattened [R',SR,K] order of sample_pidx >= 0, colour rows per
    sample slot.  Candidate s of the frustum query is entry s of the [R',SR] slots, and a valid sample's neighbours are its first K
    slots, so pair row (vi, k) is flat entry valid_list[vi] * K + k."""
    import ctypes
    from oracle import forward_check
    from pointnerf_b200 import lib
    S, P = int(q.counters["n_valid"]), int(q.counters["n_pairs"])
    out = (ctypes.c_void_p * 10)()
    ws = net._bwd_ws
    F_ = int(net.neural_points.points_embeding.shape[-1])
    lib.check(lib.load().pnb_backward_tables(ws.data_ptr(), ws.numel(), S, q.desc.cap_samples, F_, out), "pnb_backward_tables")
    dv = forward_check.dev_view
    H = [dv(ws, out[0], torch.float32, (P, 256)), dv(ws, out[1], torch.float32, (P, 272))[:, :256],
         dv(ws, out[2], torch.float32, (P, 256)), dv(ws, out[3], torch.float32, (P, 256))]
    Cc = [dv(ws, out[i], torch.float32, (S, 128)) for i in (4, 5, 6)]
    pair_off = dv(ws, out[7], torch.int32, (S + 1,)).long()
    row_samp = dv(ws, out[8], torch.int32, (P,)).long()
    vlist = dv(q.ws, q.desc.valid_list, torch.int32, (S,)).long()
    flat = vlist[row_samp] * q.K + (torch.arange(P, device=row_samp.device) - pair_off[row_samp])
    order = torch.argsort(flat)
    slopes = [torch.where(h[order] > 0, 1.0, 0.01).double().cpu() for h in H]
    for c in Cc:
        sl = torch.ones(q.R2 * q.SR, 128, dtype=torch.float64)
        sl[vlist.cpu()] = torch.where(c > 0, 1.0, 0.01).double().cpu()
        slopes.append(sl)
    return slopes


# ------------------------------------------------------------------------------------------------ conditioning of alpha_branch.0
class SoftplusInputs:
    """Stands in for torch.nn.functional in this module (recording_softplus): keeps the inputs of softplus with their gradients."""

    def __init__(self, functional):
        self._f, self.inputs = functional, []

    def __getattr__(self, k):
        return getattr(self._f, k)

    def softplus(self, x, *a, **k):
        if x.requires_grad:
            x.retain_grad()
        self.inputs.append(x)
        return self._f.softplus(x, *a, **k)


@contextlib.contextmanager
def recording_softplus():
    """shade() inside the block records its softplus inputs (the last one: sigma's pre-activation with agg_intrp_order 1)."""
    global F
    rec = SoftplusInputs(F)
    F = rec
    try:
        yield rec
    finally:
        F = rec._f


def alpha_branch_abs_terms(rec, hbar):
    """After backward() of a loss on a recorded order-1 shade(): alpha_branch.0's gradient is a sum over samples of dL/dz [1, h-bar]
    (z = alpha_branch(h-bar) - 1).  Returns {name: sum of |terms|} per entry, for grad_check.sum_error."""
    gz = rec.inputs[-1].grad.reshape(-1, 1).abs()
    return {"alpha_branch.0.bias": gz.sum(0), "alpha_branch.0.weight": (gz * hbar.detach().abs()).sum(0, keepdim=True)}
