"""GPU: the persistent tile loop of the pair and colour kernels (a producer warp runs the weight ring for the CTA's whole tile
sequence) for every kernel variant, and frames where the producer has nothing or almost nothing to do."""
import numpy as np
import pytest
import torch

from oracle import pipeline
from pointnerf_b200 import harness, lib, scene

pytestmark = pytest.mark.gpu
DEV = "cuda:0"
TOL = 1e-4
FEW_CTAS = 8          # pnb_dbg_flags bit 3: one CTA per 8 SMs, so every CTA runs many tiles


def _render_full(net, cfg, rays):
    with torch.no_grad():
        return net.render_full(list(cfg.campos), rays["raydir"].to(DEV), torch.eye(3), cfg.near, cfg.far, [1., 1., 1.])


def _set_frames(net, R):
    p = net.neural_points
    p.set_points(p.xyz.detach().clone(), p.points_embeding.detach().clone(), points_color=p.points_color.detach().clone(),
                 points_dir=p.points_dir.detach().clone(), points_conf=p.points_conf.detach().clone(), Rw2c=R.to(DEV))


def _oracle_render(cfg, opt, pts, agg, raydir):
    return pipeline.render(pts, harness.mlp_cpu(agg), raydir, cfg.campos, np.eye(3, dtype=np.float32), cfg.near, cfg.far,
                           opt.vsize, opt.vscale, opt.kernel_size, opt.query_size, opt.ranges, opt.SR, opt.K, opt.P,
                           opt.max_o if opt.max_o is not None else pts["xyz"].shape[0], D=cfg.D)


KEYS = ("coarse_raycolor", "coarse_point_opacity", "coarse_is_background")


@pytest.mark.parametrize("over,frames", [
    (dict(pnb_frozen=0), False),                                  # general kernel
    (dict(agg_intrp_order=1), False),                             # order 1, frozen
    (dict(agg_intrp_order=1, pnb_frozen=0), False),
    ({}, True),                                                   # per-point frames, frozen
    (dict(pnb_frozen=0), True),
    (dict(feat_dim=63), False),                                   # F = 63, frozen
    (dict(feat_dim=63, pnb_frozen=0), False),                     # F = 63, layer 1 in two halves
], ids=["general", "order1", "order1-general", "rw2c", "rw2c-general", "f63", "f63-general"])
def test_persistent_tile_loop_is_bit_identical_per_variant(over, frames):
    """Each k_shade_wg instantiation (and k_color_wg with and without per-point frames) on one CTA per 8 SMs against the default
    launch (one CTA per SM): the same arithmetic per tile -> equal bits."""
    cfg = scene.CONFIGS["tiny"]
    a, pts, _ = harness.build_model(cfg, DEV, alpha_bias=3.0, **over)
    b, _, _ = harness.build_model(cfg, DEV, alpha_bias=3.0, pnb_dbg_flags=FEW_CTAS, **over)
    if frames:
        R = scene.edit_frames(pts["xyz"])
        _set_frames(a, R)
        _set_frames(b, R)
    rays = scene.make_rays(cfg, scene.centre_patch(cfg, 64))
    for rep in range(2):
        oa, ob = _render_full(a, cfg, rays), _render_full(b, cfg, rays)
        a.check_errors(); b.check_errors()
        for k in KEYS:
            assert torch.equal(oa[k], ob[k]), k
    assert oa["coarse_point_opacity"].max().item() > 0.0


@pytest.mark.parametrize("dbg", [0, FEW_CTAS])
@pytest.mark.parametrize("case", ["all-miss", "few-tiles"])
def test_nearly_empty_frames_match_oracle(case, dbg):
    """A frame where no ray meets a point (no tile: the producer has no weight stage to load) and a 4 x 4 patch (a handful of
    tiles, fewer than CTAs): no error flag, the oracle's outputs."""
    cfg = scene.CONFIGS["tiny"]
    net, pts, opt = harness.build_model(cfg, DEV, alpha_bias=3.0, pnb_dbg_flags=dbg)
    rays = scene.make_rays(cfg, scene.centre_patch(cfg, 4 if case == "few-tiles" else 16))
    if case == "all-miss":
        rays["raydir"] = -rays["raydir"]                          # looking away from the cloud
    out = _render_full(net, cfg, rays)
    net.check_errors()
    ref = _oracle_render(cfg, opt, pts, net.aggregator, rays["raydir"][0])
    assert np.array_equal(out["ray_mask"][0].cpu().numpy(), ref["ray_mask"])
    for k in KEYS:
        d = (out[k][0].cpu() - ref[k]).abs().max().item()
        assert d <= TOL, "%s max abs diff %.3e" % (k, d)
    opacity = out["coarse_point_opacity"].max().item()
    assert opacity == 0.0 if case == "all-miss" else opacity > 0.0
    n_valid = int(net.last.counters_tensor()[lib.QC["n_valid"]].item())
    if case == "few-tiles":      # every 32-row quadrant holds >= 1 valid sample: tiles <= n_valid / 4 (<= 16 rays x SR / 4 = 96)
        assert 0 < (n_valid + 3) // 4 < torch.cuda.get_device_properties(0).multi_processor_count
    else:
        assert n_valid == 0
