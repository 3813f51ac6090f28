"""TEST INFRASTRUCTURE ONLY -- the whole reference path for one call, assembled from the oracle parts:
host hyper-parameters (point_query.py:47-71) -> t table (diff_ray_marching.py:349-392) ->
C query (query_oracle.c) -> shading/compositing (shade_oracle.py) -> fill_invalid.
Used by tests/ (as the checker), __graft_entry__.smoke() and bench.py's CPU-baseline legs only.
"""
import numpy as np
import torch

from . import query_oracle, shade_oracle


def hyperparameters(xyz, vsize, vscale, kernel_size, ranges):
    """point_query.py:35-42,47-71 restated with numpy's promotion rules made explicit.
    xyz: torch [N,3] f32.  Returns ranges6 (f32 np[6]), scaled_vsize (f32 np[3]), scaled_vdim (i32 np[3])."""
    vscale_np = np.array(vscale, dtype=np.int32)
    scaled_vsize_np = (np.asarray(vsize, dtype=np.float64) * vscale_np).astype(np.float32)   # :36
    mn, mx = torch.min(xyz, dim=-2)[0], torch.max(xyz, dim=-2)[0]
    if ranges is not None:
        mn = torch.maximum(mn, torch.as_tensor(ranges[:3], dtype=torch.float32))
        mx = torch.minimum(mx, torch.as_tensor(ranges[3:], dtype=torch.float32))
    pad = torch.as_tensor(scaled_vsize_np * np.asarray(kernel_size) / 2, dtype=torch.float32)  # :63 (f64 -> f32)
    mn = mn - pad
    mx = mx + pad
    vdim = (mx - mn).numpy() / np.asarray(vsize, dtype=np.float64)                             # :68
    scaled_vdim = np.ceil(vdim / vscale_np).astype(np.int32)                                   # :69
    return torch.cat([mn, mx]).numpy(), scaled_vsize_np, scaled_vdim


def t_table(near, far, D):
    """Eval-mode (jitter == 0) mid-point table of near_far_linear_ray_generation
    (diff_ray_marching.py:369-385), computed with the same fp32 torch-CPU ops."""
    tvals = torch.linspace(0, 1, D + 1).view(1, -1)
    tvals = near * (1 - tvals) + far * tvals
    seg = (tvals[..., 1:] - tvals[..., :-1]) * (1 + 0.0 * (torch.zeros(1, 1, D) - 0.5))
    end = torch.cumsum(seg, dim=2)
    end = torch.cat([torch.zeros(1, 1, 1), end], dim=2)
    end = near + end
    return ((end[:, :, :-1] + end[:, :, 1:]) / 2).reshape(D).numpy()


def radius_limit(radius_limit_scale, vsize):
    return np.asarray(radius_limit_scale * max(vsize[0], vsize[1])).astype(np.float32)   # point_query.py:35


def render(points, mlp, raydir, campos, camrotc2w, near, far, vsize, vscale, kernel_size, query_size,
           ranges, SR, K, P, max_o, D=400, radius_limit_scale=4.0, bg_color=(1., 1., 1.), t=None,
           dtype=torch.float32, want_shade=True, agg_intrp_order=2, raydist_mode_unit=1):
    """raydir [R,3] torch f32.  Returns dict: query outputs + shade outputs + fill_invalid outputs + counters."""
    rng6, svs, dim = hyperparameters(points["xyz"], vsize, vscale, kernel_size, ranges)
    if t is None:
        t = t_table(float(near), float(far), D)
    q = query_oracle.query(points["xyz"].numpy(), rng6[:3], svs, dim, kernel_size, query_size, max_o, P,
                           float(radius_limit(radius_limit_scale, vsize)),
                           campos=np.asarray(campos, np.float32), raydir=raydir.numpy(), t=t, SR=SR, K=K)
    out = dict(q)
    out.update(ranges6=rng6, scaled_vsize=svs, scaled_vdim=dim, t=np.asarray(t))
    if not want_shade:
        return out
    mask = torch.from_numpy(q["ray_mask"]) > 0
    if int(mask.sum()) == 0:
        # no ray keeps a neighbour: the reference returns empty R' tensors (neural_points_volumetric_model.py:352-361) and fill_invalid
        # paints the whole chunk with the background
        R = mask.shape[0]
        bg = torch.as_tensor(bg_color).to(dtype)
        out.update(ray_color=torch.zeros(0, 3, dtype=dtype), opacity=torch.zeros(0, SR, dtype=dtype), bg_T=torch.zeros(0, 1, dtype=dtype),
                   coarse_raycolor=torch.ones(R, 3, dtype=dtype) * bg.view(1, 3), coarse_is_background=torch.ones(R, 1, dtype=dtype),
                   coarse_mask=torch.zeros(R, 1, dtype=dtype), coarse_point_opacity=torch.zeros(R, SR, dtype=dtype),
                   queried_shading=torch.ones(R, 3, dtype=dtype))
        return out
    sh = shade_oracle.shade(points, mlp, torch.from_numpy(q["sample_pidx"]), torch.from_numpy(q["sample_loc_w"]),
                            raydir[mask], torch.as_tensor(campos), torch.as_tensor(camrotc2w), vsize,
                            torch.as_tensor(bg_color), dtype=dtype, agg_intrp_order=agg_intrp_order, raydist_mode_unit=raydist_mode_unit)
    out.update(sh)
    out.update(shade_oracle.fill_invalid(mask, sh["ray_color"], sh["opacity"], sh["bg_T"], sh["queried_shading"],
                                         torch.as_tensor(bg_color)))
    return out
