"""TEST INFRASTRUCTURE ONLY -- generates tests/golden/tiny_rw2c by running the reference's OWN, unmodified Python hot path on CPU
(the build of oracle/make_golden.py) on a point cloud with per-point frames, neural_points.Rw2c [N,3,3]:

    python -m oracle.make_golden_rw2c

The case is tiny_opaque's (tiny scene, 40x40 centre patch, alpha bias 4, SR 24) with the frames of an edit (scene.edit_frames: the
cloud split by sign(x) into two objects, each rotated about a different axis), stored as NeuralPoints.set_points stores a supplied
Rw2c (neural_points.py:463-467).  The fixture holds what golden_case stores for the uniform cases plus the frames (key Rw2c); the
loss of the gradients is the same.  It pins oracle/shade_oracle_rw2c.py (tests/test_rw2c.py) and the CUDA path
(tests/test_gpu_rw2c.py).
"""
import os
import sys

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

from oracle import golden, query_oracle, ref_shim  # noqa: E402
from oracle.make_golden import OUT, build_reference_net  # noqa: E402
from pointnerf_b200 import scene  # noqa: E402


def golden_case_rw2c(name, cfg, pixels, alpha_bias, SR=24):
    net, agg, npts, pts, opt = build_reference_net(cfg, alpha_bias, SR=SR)
    npts.Rw2c = torch.nn.Parameter(scene.edit_frames(npts.xyz.detach()), requires_grad=False)
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
        grad_embedding=g["neural_points.points_embeding"].numpy(), grad_color=g["neural_points.points_color"].numpy(),
        grad_dir=g["neural_points.points_dir"].numpy(), grad_conf=g["neural_points.points_conf"].numpy(),
        Rw2c=npts.Rw2c.detach().numpy(),
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
    golden_case_rw2c("tiny_rw2c", tiny, scene.centre_patch(tiny, 40), alpha_bias=4.0)
