"""CPU checks for shading the perspective-frustum query in the fused module (wcoord_query 0): the float64 restatement its GPU checks
use (tests/frustum_shade_f64.py: agg_intrp_order 1 and 2, given LeakyReLU masks, per-sample outputs) against oracle/shade_oracle_frustum.py
and oracle/shade_oracle.py, which options the fused module accepts with that query, and the host-side bg_ray fill of the chunked
whole-image loop against the reference's fill_invalid."""
import numpy as np
import pytest
import torch

import frustum_shade_f64
from oracle import frustum_oracle, shade_oracle, shade_oracle_frustum
from pointnerf_b200 import harness
from pointnerf_b200 import query_point_indices as qpi
from pointnerf_b200 import scene


def _oracle_query(pixels):
    cfg = scene.FRUSTUM_CONFIGS["dtu_surface"]
    s = scene.make_frustum_scene(cfg)
    opt = scene.frustum_opt(cfg)
    rl, dl, ranges, vsize, vdim, svs, sdim, vscale = qpi.hyperparameters(opt, np.int64(cfg.H), np.int64(cfg.W), s["intrinsic"],
                                                                         np.float32(cfg.near), np.float32(cfg.far))
    out = frustum_oracle.query(s["pers"], ranges[:3], svs, sdim, vscale, opt.kernel_size, opt.query_size, opt.SR, opt.K, opt.P,
                               pixels, np.float32(rl ** 2), np.float32(dl ** 2), max_o=opt.max_o)
    return cfg, s, opt, out


def _case(stride, seed):
    from pointnerf_b200.ray_marching import PointAggregator
    cfg = scene.FRUSTUM_CONFIGS["dtu_surface"]
    _, s, opt, out = _oracle_query(scene.make_frustum_scene(cfg)["pixel_idx"][::stride])
    pts = scene.make_frustum_points(cfg, s)
    mlp = {k: v.detach() for k, v in PointAggregator(harness.make_opt(scene.CONFIGS["tiny"], feat_dim=63), seed=seed).state_dict().items()}
    rot, pos = torch.from_numpy(s["camrotc2w"]), torch.from_numpy(s["campos"])
    return opt, pts, mlp, rot, pos, out


def _random_slopes(pidx, SR, seed):
    """Per-unit slopes (1 or 0.01) of the 7 LeakyReLU layers in the layout of oracle/shade_oracle.py's `slopes=`."""
    g = torch.Generator().manual_seed(seed)
    P, S = int((pidx >= 0).sum()), pidx.shape[0] * SR
    pick = lambda n, c: torch.where(torch.rand(n, c, generator=g) > 0.3, 1.0, 0.01).double()  # noqa: E731
    return [pick(P, 256) for _ in range(4)] + [pick(S, 128) for _ in range(3)]


@pytest.mark.parametrize("dtype", [torch.float32, torch.float64])
def test_restatement_matches_shade_oracle_frustum(dtype):
    """On the frustum query's own tuple, tests/frustum_shade_f64.py with its defaults (order 2, LeakyReLU) computes exactly what
    oracle/shade_oracle_frustum.py computes."""
    opt, pts, mlp, rot, pos, out = _case(40, 3)
    loc = torch.from_numpy(out["sample_loc"])
    loc_w, dirs = qpi.lighting_fast_querier.pers2w(None, loc[None], rot[None], pos[None])
    args = (pts, mlp, torch.from_numpy(out["sample_pidx"]), loc, loc_w[0], dirs[0], pos, rot, (0.005, 0.005, 0.0068125), torch.ones(3))
    a = shade_oracle_frustum.shade(*args, dtype=dtype)
    b = frustum_shade_f64.shade(*args, dtype=dtype)
    assert (a["opacity"] > 0).any()
    for k in ("ray_color", "opacity", "bg_T"):
        assert torch.equal(a[k], b[k]), k


@pytest.mark.parametrize("masks", [False, True])
@pytest.mark.parametrize("order", [1, 2])
def test_restatement_order_and_slopes_match_shade_oracle(order, masks):
    """Given the world query's per-sample inputs (sample_loc = w2pers(sample_loc_w), one direction per ray), the restatement with
    agg_intrp_order=order and slopes= computes exactly what oracle/shade_oracle.py computes with them, decoded (sigma, rgb) included
    (the method of test_oracle_frustum's order-2 check)."""
    opt, pts, mlp, rot, pos, out = _case(40, 3)
    loc_w, dirs = qpi.lighting_fast_querier.pers2w(None, torch.from_numpy(out["sample_loc"])[None], rot[None], pos[None])
    loc_w, ray_dir = loc_w[0], dirs[0, :, 0]
    pidx = torch.from_numpy(out["sample_pidx"])
    vsize = (0.005, 0.005, 0.0068125)
    slopes = _random_slopes(pidx, opt.SR, 7) if masks else None
    a = shade_oracle.shade(pts, mlp, pidx, loc_w, ray_dir, pos, rot, vsize, torch.ones(3), dtype=torch.float64, agg_intrp_order=order,
                           slopes=slopes)
    b = frustum_shade_f64.shade(pts, mlp, pidx, shade_oracle.w2pers(loc_w.double(), rot.double(), pos.double()), loc_w,
                                ray_dir[:, None, :].expand(-1, opt.SR, -1), pos, rot, vsize, torch.ones(3), agg_intrp_order=order,
                                slopes=slopes)
    assert pidx.shape[0] > 100 and (a["opacity"] > 0).any()
    for k in ("ray_color", "opacity", "bg_T", "decoded"):
        assert torch.equal(a[k], b[k]), k
    if masks:   # the masks reach the result
        c = frustum_shade_f64.shade(pts, mlp, pidx, shade_oracle.w2pers(loc_w.double(), rot.double(), pos.double()), loc_w,
                                    ray_dir[:, None, :].expand(-1, opt.SR, -1), pos, rot, vsize, torch.ones(3), agg_intrp_order=order)
        assert not torch.equal(b["decoded"], c["decoded"])


def _frustum_model_opt(**over):
    return harness.make_opt(scene.CONFIGS["tiny"], feat_dim=63, wcoord_query=0, **over)


def test_check_opt_accepts_the_dtu_frustum_configuration():
    from pointnerf_b200.ray_marching import check_opt
    check_opt(_frustum_model_opt())
    check_opt(_frustum_model_opt(agg_intrp_order=1))


@pytest.mark.parametrize("over", [dict(feat_dim=32), dict(point_conf_mode="1"), dict(point_dir_mode="1"), dict(point_color_mode="1"),
                                  dict(NN=1), dict(NN=0), dict(raydist_mode_unit=0)])
def test_check_opt_refuses_the_frustum_query_outside_the_dtu_configuration(over):
    from pointnerf_b200.ray_marching import check_opt
    fd = over.pop("feat_dim", 63)
    opt = harness.make_opt(scene.CONFIGS["tiny"], feat_dim=fd, wcoord_query=0, **over)
    with pytest.raises(NotImplementedError, match="wcoord_query=0"):
        check_opt(opt)


def test_chunk_fill_with_bg_ray_is_the_reference_fill_invalid():
    """runner's per-chunk bg_ray fill is the model shell's fill_invalid (neural_points_volumetric_model.py:87-103) on B = 1."""
    from pointnerf_b200.runner import _fill_bg_ray
    g = torch.Generator().manual_seed(0)
    R = 257
    mask = torch.rand(R, generator=g) > 0.4
    n = int(mask.sum())
    color, is_bg, bg_ray = torch.rand(n, 3, generator=g), torch.rand(n, 1, generator=g), torch.rand(R, 3, generator=g)
    ours = _fill_bg_ray(color, is_bg, mask, bg_ray)
    # the reference's statements, [B, OR, ...] with B = 1
    ray_inds = torch.nonzero(mask[None])
    cib = torch.ones([1, R, 1])
    cib[ray_inds[..., 0], ray_inds[..., 1], :] = is_bg[None]
    want = cib * bg_ray[None]
    want[ray_inds[..., 0], ray_inds[..., 1], :] += color
    assert torch.equal(ours, want[0])
