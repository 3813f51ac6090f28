"""Build the hot-path modules for one of the synthetic BASELINE configs (used by tests/, bench.py, smoke())."""
from types import SimpleNamespace

import torch

from . import scene
from .ray_marching import NeuralPoints, NeuralPointsRayMarching, PointAggregator


def make_opt(cfg, is_train=False, feat_dim=32, **over):
    """The option surface the hot path reads (SURVEY.md 8b), with the shipped values (section 8 head).  feat_dim 63: the DTU
    scripts' point_features_dim 63 with point_{conf,dir,color}_mode "01"."""
    o = SimpleNamespace(
        # querier (point_query.py:33-42,76-93)
        inverse=0, radius_limit_scale=cfg.radius_limit_scale, vsize=[cfg.vsize] * 3, vscale=[cfg.vscale] * 3,
        kernel_size=[cfg.kernel_size] * 3, query_size=[cfg.query_size] * 3, ranges=list(scene.ranges_for(cfg)),
        z_depth_dim=cfg.D, is_train=is_train, SR=cfg.SR, K=cfg.K, max_o=None, P=cfg.P, gpu_maxthr=1024, NN=2,
        # NeuralPoints
        wcoord_query=-1, load_points=0, point_features_dim=32, xyz_grad=0, feat_grad=1, conf_grad=1, color_grad=1,
        dir_grad=1, default_conf=-1.0, point_conf_mode="1", point_dir_mode="1", point_color_mode="1",
        # aggregator
        act_type="LeakyReLU", agg_distance_kernel="linear", agg_dist_pers=20, agg_axis_weight=None,
        num_pos_freqs=10, num_viewdir_freqs=4, view_ori=0, which_agg_model="viewmlp", agg_intrp_order=2,
        apply_pnt_mask=1, dist_xyz_deno=0, dist_xyz_freq=5, num_feat_freqs=3, agg_feat_xyz_mode="None",
        agg_alpha_xyz_mode="None", agg_color_xyz_mode="None", shading_feature_mlp_layer1=2,
        shading_feature_mlp_layer2=0, shading_feature_mlp_layer3=2, shading_feature_num=256,
        shading_alpha_mlp_layer=1, shading_color_mlp_layer=4, shading_color_channel_num=3, act_super=1,
        agg_weight_norm=1, sparse_loss_weight=0, zero_one_loss_items=["conf_coefficient"], prob=0,
        # ray marcher
        raydist_mode_unit=1, which_render_func="radiance", which_blend_func="alpha", which_tonemap_func="off",
    )
    if feat_dim != 32:
        o.point_features_dim = feat_dim
        o.point_conf_mode = o.point_dir_mode = o.point_color_mode = "01"
    for k, v in over.items():
        setattr(o, k, v)
    return o


def build_model(cfg, device, seed=0, alpha_bias=0.0, is_train=False, feat_dim=32, **over):
    """Returns (net, points_cpu_dict, opt).  MLP init seed `seed`; alpha_bias raises alpha_branch.0.bias
    to make the scene opaque (a more discriminating parity case, SURVEY section 7).  feat_dim 63: the DTU configuration (56 image
    features, colour, dir and conf prepended by set_points)."""
    opt = make_opt(cfg, is_train=is_train, feat_dim=feat_dim, **over)
    pts = scene.make_points(cfg, emb_dim=32 if feat_dim == 32 else feat_dim - 7)
    agg = PointAggregator(opt, seed=seed)
    with torch.no_grad():
        agg.alpha_branch[0].bias += alpha_bias
    agg = agg.to(device)
    npnts = NeuralPoints(opt, device)
    npnts.set_points(pts["xyz"].to(device), pts["embedding"].to(device), points_color=pts["color"].to(device),
                     points_dir=pts["dir"].to(device), points_conf=pts["conf"].to(device), parameter=True)
    net = NeuralPointsRayMarching(aggregator=agg, neural_points=npnts, opt=opt)
    return net, pts, opt


def mlp_cpu(agg):
    return {k: v.detach().cpu() for k, v in agg.state_dict().items()}
