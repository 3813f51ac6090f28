"""TEST INFRASTRUCTURE ONLY (imported by tests/test_oracle_frustum_fused.py and tests/test_gpu_frustum_fused.py; not a test module).

The reference's eager shading of a perspective-frustum query result, as oracle/shade_oracle_frustum.py restates it, with what the
fused-module checks need beyond that restatement:
  agg_intrp_order  2 (alpha per neighbour, then the weighted sum) or 1 (alpha_branch on the K-aggregated feature,
                   point_aggregators.py:573-587), as oracle/shade_oracle.py takes it
  slopes           None (LeakyReLU) or the per-unit slopes of the 7 LeakyReLU layers (another computation's masks), as
                   oracle/shade_oracle.py takes them
  decoded          (sigma, rgb) of every sample [R',SR,4] in the result, for the per-sample comparison of DESIGN.md §6 item 6
tests/test_oracle_frustum_fused.py holds it bit for bit to oracle/shade_oracle_frustum.shade (order 2, no slopes) on the frustum
query's tuple and to oracle/shade_oracle.shade (orders 1 and 2, with and without slopes) on the world query's inputs.
"""
import torch
import torch.nn.functional as F

from oracle.shade_oracle import _act, _lin, positional_encoding, w2pers


def shade(points, mlp, sample_pidx, sample_loc, sample_loc_w, sample_ray_dirs, campos, camrotc2w, vsize, bg_color, dtype=torch.float64,
          agg_intrp_order=2, slopes=None):
    """Arguments as oracle/shade_oracle_frustum.shade (the querier's tuple without the batch dimension; vsize: the querier's).
    Returns dict(ray_color [R',3], opacity [R',SR], bg_T [R',1], decoded [R',SR,4])."""
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
    wc = weight * (c0 - (c0 - torch.clamp(c0, min=0.0001, max=1)).detach())
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

    # ray distances (neural_points_volumetric_model.py:271-279) and ray_march (diff_ray_marching.py:508-554)
    vz = float(vsize[2])
    z = torch.cummax(sample_loc[..., 2], dim=-1)[0]
    ray_dist = torch.cat([z[..., 1:] - z[..., :-1], torch.full((Rn, 1), vz, dtype=dtype)], dim=-1)
    m = torch.logical_or(ray_dist < 1e-8, ray_dist > 2 * vz).to(dtype)
    ray_dist = (ray_dist * (1.0 - m) + m * vz) * ray_valid.to(dtype)
    opacity = 1 - torch.exp(-decoded[..., 0] * ray_valid.to(dtype) * ray_dist)
    acc = torch.cumprod(1. - opacity + 1e-10, dim=-1)
    bg_T = acc[:, -1:]
    acc_T = torch.cat([torch.ones(Rn, 1, dtype=dtype), acc[:, :-1]], dim=-1)
    ray_color = torch.sum(decoded[..., 1:4] * (opacity * acc_T)[..., None], dim=-2) + bg_color.view(1, 3) * bg_T
    return dict(ray_color=ray_color, opacity=opacity, bg_T=bg_T, decoded=decoded)
