"""TEST INFRASTRUCTURE ONLY -- CPU restatement (torch, eager) of the reference's per-sample shading + compositing for a point cloud
with one world->canonical rotation per point, neural_points.Rw2c [N,3,3] (edited / composed scenes, run/editing.py:186-212).

The same computation as oracle/shade_oracle.py, whose helpers it uses, with the reference's per-point ops
(models/aggregators/point_aggregators.py:491-496, :506, :526, :566; gather models/neural_points/neural_points.py:717):
  dists[0:3] and the point direction are rotated into the frame of the pair's own point,
  the view direction (PE(view) and the view extras of every pair of the sample) into the frame of the sample's slot-0 neighbour,
each as the reference's batched `[..., 1, 3] @ [..., 3, 3]` product of the transposed gathered frames, so the forward matches the
reference bit for bit (tests/test_rw2c.py against tests/golden/tiny_rw2c, written by oracle/make_golden_rw2c.py).  A uniform [3,3]
Rw2c is handed to shade_oracle.shade unchanged.  Differentiable: autograd through `shade()` is the backward oracle.
"""
import torch
import torch.nn.functional as F

from .shade_oracle import LEAKY_SLOPE, _act, _lin, fill_invalid, positional_encoding, w2pers  # noqa: F401  (fill_invalid: re-exported)
from . import shade_oracle


def shade(points, mlp, sample_pidx, sample_loc_w, raydir_hit, campos, camrotc2w, vsize, bg_color,
          dtype=torch.float32, agg_intrp_order=2, slopes=None, raydist_mode_unit=1):
    """The arguments and the returned dict of shade_oracle.shade; points["Rw2c"] is [3,3] or [N,3,3]."""
    if points["Rw2c"].dim() == 2:
        return shade_oracle.shade(points, mlp, sample_pidx, sample_loc_w, raydir_hit, campos, camrotc2w, vsize, bg_color,
                                  dtype=dtype, agg_intrp_order=agg_intrp_order, slopes=slopes, raydist_mode_unit=raydist_mode_unit)
    assert agg_intrp_order in (1, 2)
    cv = lambda t: t.to(dtype)
    xyz = cv(points["xyz"]); emb = cv(points["embedding"][0]); col = cv(points["color"][0])
    pdir = cv(points["dir"][0]); conf = cv(points["conf"][0]); Rw2c = cv(points["Rw2c"])
    assert Rw2c.shape == (xyz.shape[0], 3, 3)
    mlp = {k: cv(v) for k, v in mlp.items()}
    sample_loc_w = cv(sample_loc_w); raydir_hit = cv(raydir_hit)
    campos = cv(campos).reshape(3); camrotc2w = cv(camrotc2w).reshape(3, 3); bg_color = cv(bg_color).reshape(3)
    Rn, SR, K = sample_pidx.shape

    # ---- gather (neural_points.py:706-717) ----
    pnt_mask = sample_pidx >= 0
    idx = torch.clamp(sample_pidx, min=0).reshape(-1).long()
    xyz_pers_all = w2pers(xyz, camrotc2w, campos)
    s_xyz = xyz[idx].view(Rn, SR, K, 3)
    s_xyz_pers = xyz_pers_all[idx].view(Rn, SR, K, 3)
    s_emb = emb[idx].view(Rn, SR, K, -1)
    s_col = col[idx].view(Rn, SR, K, 3)
    s_dir = pdir[idx].view(Rn, SR, K, 3)
    s_conf = conf[idx].view(Rn, SR, K, 1)
    sRt = Rw2c[idx].view(Rn, SR, K, 3, 3).transpose(-1, -2)          # :717, transposed as viewmlp does (:492)
    sample_loc = w2pers(sample_loc_w, camrotc2w, campos)
    sample_ray_dirs = raydir_hit[:, None, :].expand(-1, SR, -1)

    # ---- PointAggregator.forward (point_aggregators.py:727-814), agg_dist_pers == 20 ----
    ray_valid = torch.any(pnt_mask, dim=-1)
    xdist = s_xyz_pers[..., 0] * s_xyz_pers[..., 2] - sample_loc[:, :, None, 0] * sample_loc[:, :, None, 2]
    ydist = s_xyz_pers[..., 1] * s_xyz_pers[..., 2] - sample_loc[:, :, None, 1] * sample_loc[:, :, None, 2]
    zdist = s_xyz_pers[..., 2] - sample_loc[:, :, None, 2]
    dists = torch.cat([s_xyz - sample_loc_w[..., None, :], torch.stack([xdist, ydist, zdist], dim=-1)], dim=-1)
    weight = pnt_mask * (1.0 / torch.clamp(torch.norm(dists[..., :3], dim=-1), min=1e-6))
    weight = weight / torch.clamp(torch.sum(weight, dim=-1, keepdim=True), min=1e-8)
    c0 = s_conf[..., 0]
    conf_coefficient = c0 - (c0 - torch.clamp(c0, min=0.0001, max=1)).detach()
    wc = weight * conf_coefficient

    # ---- viewmlp (point_aggregators.py:488-644) with per-point frames ----
    pm = pnt_mask.reshape(-1)
    Rt_ray = sRt[:, :, 0, :, :].reshape(-1, 3, 3)                      # the sample's slot-0 neighbour (:495)
    Rt_pair = sRt.reshape(-1, 3, 3)[pm]                                # the pair's own point (:496)
    rot_view = lambda v: (v[..., None, :] @ Rt_ray).squeeze(-2)        # :506
    rot_pair = lambda v: (v[..., None, :] @ Rt_pair).squeeze(-2)       # :526, :566
    viewdirs = rot_view(sample_ray_dirs.reshape(-1, 3))
    pe_view = positional_encoding(viewdirs, 4, ori=True)
    ori_viewdirs, pe_view = pe_view[..., :3], pe_view[..., 3:]
    sv = ray_valid.reshape(-1)
    d_flat = dists.reshape(-1, 6)[pm]
    d_flat = torch.cat([rot_pair(d_flat[:, :3]), d_flat[:, 3:]], dim=-1)
    d_pe = positional_encoding(d_flat, 5)
    f = s_emb.reshape(-1, s_emb.shape[-1])[pm]
    feat = torch.cat([f, positional_encoding(f, 3), d_pe], dim=-1)
    act = lambda x, layer: _act(x, slopes, layer)
    feat = act(_lin(act(_lin(feat, mlp, "block1.0"), 0), mlp, "block1.2"), 1)
    c_flat = s_col.reshape(-1, 3)[pm]
    dir_flat = rot_pair(s_dir.reshape(-1, 3)[pm])
    ov = ori_viewdirs[:, None, :].expand(-1, K, -1).reshape(-1, 3)[pm]
    feat = torch.cat([feat, c_flat, dir_flat - ov, torch.sum(dir_flat * ov, dim=-1, keepdim=True)], dim=-1)
    feat = act(_lin(act(_lin(feat, mlp, "block3.0"), 2), mlp, "block3.2"), 3)
    alpha = F.softplus(_lin(feat, mlp, "alpha_branch.0") - 1)
    n_pair = Rn * SR * K
    pm_idx = pm.nonzero()[:, 0]
    alpha_h = torch.zeros(n_pair, 1, dtype=dtype).index_put((pm_idx,), alpha)
    feat_h = torch.zeros(n_pair, feat.shape[-1], dtype=dtype).index_put((pm_idx,), feat)
    wflat = wc.reshape(Rn * SR, K, 1)
    hbar = torch.sum(feat_h.view(Rn * SR, K, -1) * wflat, dim=-2)
    if agg_intrp_order == 2:
        sigma = torch.sum(alpha_h.view(Rn * SR, K, 1) * wflat, dim=-2)
    else:
        sigma = F.softplus(_lin(hbar, mlp, "alpha_branch.0") - 1)
    cin = torch.cat([hbar, pe_view], dim=-1)
    x = act(_lin(cin, mlp, "color_branch.0"), 4)
    x = act(_lin(x, mlp, "color_branch.2"), 5)
    x = act(_lin(x, mlp, "color_branch.4"), 6)
    rgb = torch.sigmoid(_lin(x, mlp, "color_branch.6")) * (1 + 2 * 0.001) - 0.001
    decoded = torch.cat([sigma, rgb], dim=-1)
    decoded = torch.where(sv[:, None], decoded, torch.zeros_like(decoded))
    decoded = decoded.view(Rn, SR, 4)

    # ---- ray distances (neural_points_volumetric_model.py:271-279) ----
    vz = float(vsize[2])
    z = torch.cummax(sample_loc[..., 2], dim=-1)[0]
    ray_dist = torch.cat([z[..., 1:] - z[..., :-1], torch.full((Rn, 1), vz, dtype=dtype)], dim=-1)
    m = ray_dist < 1e-8
    if raydist_mode_unit > 0:
        m = torch.logical_or(m, ray_dist > 2 * vz)
    m = m.to(dtype)
    ray_dist = ray_dist * (1.0 - m) + m * vz
    ray_dist = ray_dist * ray_valid.to(dtype)

    # ---- ray_march (diff_ray_marching.py:508-554) ----
    sig = decoded[..., 0] * ray_valid.to(dtype)
    opacity = 1 - torch.exp(-sig * ray_dist)
    acc = torch.cumprod(1. - opacity + 1e-10, dim=-1)
    bg_T = acc[:, -1:]
    acc_T = torch.cat([torch.ones(Rn, 1, dtype=dtype), acc[:, :-1]], dim=-1)
    blend_weight = (opacity * acc_T)[..., None]
    ray_color = torch.sum(decoded[..., 1:4] * blend_weight, dim=-2) + bg_color.view(1, 3) * bg_T
    return dict(decoded=decoded, ray_valid=ray_valid, weight=weight, conf_coefficient=conf_coefficient, hbar=hbar,
                ray_dist=ray_dist, opacity=opacity, acc_T=acc_T, blend_weight=blend_weight, bg_T=bg_T,
                ray_color=ray_color, sample_loc=sample_loc,
                queried_shading=torch.logical_not(torch.any(ray_valid, dim=-1, keepdim=True)).repeat(1, 3).to(dtype))
