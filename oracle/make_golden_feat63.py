"""TEST INFRASTRUCTURE ONLY -- generates tests/golden/tiny_feat63* by running the reference's OWN, unmodified Python hot path on CPU
(the build of oracle/make_golden.py) in the DTU configuration: point_features_dim 63 with point_{conf,dir,color}_mode "01"
(dev_scripts/dtu_test_inf/inftest_scan*.sh, dev_scripts/ete/dtu_dgt_d012_img0123_conf_color_dir_agg2.sh):

    python -m oracle.make_golden_feat63

The reference's NeuralPoints.set_points gets 56 image features plus colour, dir and conf and forms the 63-channel embedding
[color, dir, conf, emb] itself (neural_points.py:401-436), keeping the three tensors as parameters of their own as well; its
PointAggregator builds block1.0 for 7 * 63 + 60 = 501 inputs (point_aggregators.py:278-280).  Cases: the tiny_opaque pixels (tiny
scene, 40x40 centre patch, alpha bias 4, SR 24) with agg_intrp_order 2 (tiny_feat63) and 1 (tiny_feat63_order1).  A fixture holds
what oracle/make_golden_rw2c.py stores (forward outputs, query, gradients of the embedding, colour, dir, conf and the 18 MLP tensors
under the loss of oracle/make_golden.py).  It pins oracle/shade_oracle.py at F = 63 (tests/test_feat63.py) and the CUDA path
(tests/test_gpu_feat63.py).
"""
import os
import sys

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

from oracle import golden, query_oracle, ref_shim  # noqa: E402
from oracle.make_golden import OUT  # noqa: E402
from pointnerf_b200 import scene  # noqa: E402

FEAT = 63
FLAGS = ("--point_features_dim", str(FEAT), "--point_conf_mode", "01", "--point_dir_mode", "01", "--point_color_mode", "01")


def build_reference_net_feat63(cfg, alpha_bias, SR=24, order=2):
    """oracle/make_golden.py:build_reference_net in the DTU configuration (it hard-codes the 32-channel cloud)."""
    ref_shim.install()
    from models.neural_points_volumetric_model import NeuralPointsRayMarching
    from models.neural_points.neural_points import NeuralPoints
    from models.aggregators.point_aggregators import PointAggregator
    from models.rendering.diff_render_func import find_render_function, find_blend_function, find_tone_map
    vs = str(cfg.vsize)
    opt = ref_shim.make_opt(["--vsize", vs, vs, vs, "--P", str(cfg.P), "--SR", str(SR), "--K", str(cfg.K),
                             "--kernel_size"] + [str(cfg.kernel_size)] * 3 + ["--query_size"] + [str(cfg.query_size)] * 3 +
                            ["--ranges"] + [str(v) for v in scene.ranges_for(cfg)] + list(FLAGS) +
                            ["--agg_intrp_order", str(order)], is_train=False)
    pts = scene.make_points(cfg, emb_dim=FEAT - 7)
    torch.manual_seed(0)
    agg = PointAggregator(opt)
    assert tuple(agg.block1[0].weight.shape) == (256, 7 * FEAT + 60)
    with torch.no_grad():
        agg.alpha_branch[0].bias += alpha_bias
    npts = NeuralPoints(FEAT, 8192, opt, torch.device("cpu"))
    npts.querier.device = "cpu"   # point_query.py:31 hard-codes "cuda"; instance attribute only, source untouched
    npts.set_points(pts["xyz"], pts["embedding"], points_color=pts["color"], points_dir=pts["dir"],
                    points_conf=pts["conf"], parameter=True)
    assert tuple(npts.points_embeding.shape) == (1, cfg.N, FEAT)
    net = NeuralPointsRayMarching(tonemap_func=find_tone_map("off"), render_func=find_render_function("radiance"),
                                  blend_func=find_blend_function("alpha"), aggregator=agg, neural_points=npts, opt=opt,
                                  num_pos_freqs=10, num_viewdir_freqs=4)
    return net, agg, npts, pts, opt


def golden_case_feat63(name, cfg, pixels, alpha_bias, SR=24, order=2):
    net, agg, npts, pts, opt = build_reference_net_feat63(cfg, alpha_bias, SR=SR, order=order)
    rays = scene.make_rays(cfg, pixels)
    out = net(rays["campos"], rays["raydir"], bg_color=rays["bg_color"], camrotc2w=rays["camrotc2w"],
              pixel_idx=rays["pixel_idx"], near=rays["near"], far=rays["far"], h=rays["h"], w=rays["w"],
              intrinsic=rays["intrinsic"])
    q = npts.querier
    rng_t, vsz, sdim = q.get_hyperparameters(opt.vsize, npts.xyz[None], ranges=opt.ranges)
    qp = q.query_points(rays["pixel_idx"].to(torch.int32), npts.w2pers(npts.xyz, rays["camrotc2w"], rays["campos"]),
                        npts.xyz[None], torch.tensor([npts.xyz.shape[0]], dtype=torch.int32), 0, 0, None,
                        np.float32(cfg.near), np.float32(cfg.far), rays["raydir"], rays["campos"], rays["camrotc2w"])
    loss = (out["coarse_raycolor"] ** 2).sum() + 1e-3 * out["conf_coefficient"].sum()
    loss.backward()
    g = {n: p.grad for n, p in net.named_parameters() if p.grad is not None}
    fx = dict(
        alpha_bias=np.float32(alpha_bias), SR=np.int32(SR), pixels=np.asarray(pixels, np.float32), agg_intrp_order=np.int32(opt.agg_intrp_order),
        ranges6=rng_t.detach().numpy(), scaled_vdim=sdim, counters=np.array([query_oracle.last_counters[k] for k in query_oracle.COUNTER_NAMES], np.int32),
        ray_mask=out["ray_mask"][0].numpy(), sample_pidx=qp[0][0].numpy(), sample_loc=qp[1][0].detach().numpy(),
        sample_loc_w=qp[2][0].numpy(),
        coarse_raycolor=out["coarse_raycolor"][0].detach().numpy(),
        coarse_point_opacity=out["coarse_point_opacity"][0].detach().numpy(),
        coarse_is_background=out["coarse_is_background"][0].detach().numpy(),
        weight=out["weight"][0].numpy(), conf_coefficient=out["conf_coefficient"][0].detach().numpy(),
        blend_weight=out["blend_weight"][0].numpy(),
        embedding63=npts.points_embeding.detach().numpy(),
        grad_embedding=g["neural_points.points_embeding"].numpy(), grad_color=g["neural_points.points_color"].numpy(),
        grad_dir=g["neural_points.points_dir"].numpy(), grad_conf=g["neural_points.points_conf"].numpy(),
    )
    for k, v in agg.state_dict().items():
        fx["mlp." + k] = v.detach().numpy()
        fx["gradmlp." + k] = g["aggregator." + k].numpy()
    os.makedirs(OUT, exist_ok=True)
    golden.save(OUT, name, fx)                                  # split into files < 1 MB (oracle/golden.py)
    print(name, "R'=%d" % fx["sample_pidx"].shape[0], "bgT mean %.3f" % fx["coarse_is_background"].mean(),
          {k: query_oracle.last_counters[k] for k in ("n_occ", "max_pts", "n_valid_samples", "n_valid_pairs")})


if __name__ == "__main__":
    assert ref_shim.available(), "needs the reference tree"
    tiny = scene.CONFIGS["tiny"]
    golden_case_feat63("tiny_feat63", tiny, scene.centre_patch(tiny, 40), alpha_bias=4.0)
    golden_case_feat63("tiny_feat63_order1", tiny, scene.centre_patch(tiny, 40), alpha_bias=4.0, order=1)
