"""GPU parity of the backward path (per-scene optimisation step): gradients of the point features and of the 18 MLP
tensors through the drop-in NeuralPointsRayMarching.forward(), against (a) gradients the reference's own autograd
produced (tests/golden, oracle/make_golden.py) and (b) autograd through oracle/shade_oracle.py on a second scene."""
import os

import numpy as np
import pytest
import torch

from oracle import pipeline, shade_oracle
from pointnerf_b200 import harness, scene
from oracle import golden  # noqa: E402

pytestmark = pytest.mark.gpu
DEV = "cuda:0"


def _close(a, ref, name, rtol=3e-4):
    a, ref = np.asarray(a, np.float64), np.asarray(ref, np.float64)
    scale = max(np.abs(ref).max(), 1e-6)
    d = np.abs(a - ref).max()
    assert d <= rtol * scale + 1e-7, "%s: max abs diff %.3e vs scale %.3e" % (name, d, scale)


def _close_points(a, ref, name, rtol=3e-4, max_outlier_frac=0.01, outlier_rtol=2e-2):
    """Per-point gradients of the tensor-core backward: its forward recompute carries the BF16x3 error, so ~1e-6 of the LeakyReLU
    units (those with a pre-activation within ~1e-5 of zero) get the other mask than the fp32 reference; each such unit changes the
    gradient of ONE pair - i.e. of one point - by ~1/256 of that pair's contribution (csrc/backward.cu header).  So: the strict tolerance on all points but <= 1 % of them (a few tens of flips per backward), and a bound on those."""
    a, ref = np.asarray(a, np.float64)[0], np.asarray(ref, np.float64).reshape(np.asarray(a).shape)[0]
    scale = max(np.abs(ref).max(), 1e-6)
    d = np.abs(a - ref).max(axis=-1)
    bad = d > rtol * scale + 1e-7
    assert bad.sum() <= max(4, max_outlier_frac * d.shape[0]), "%s: %d of %d points beyond %.0e of scale" % (name, int(bad.sum()), d.shape[0], rtol)
    assert d.max() <= outlier_rtol * scale, "%s: max abs diff %.3e vs scale %.3e" % (name, d.max(), scale)


def _forward(net, cfg, rays):
    r = {k: v.to(DEV) for k, v in rays.items()}
    return net(r["campos"], r["raydir"], bg_color=r["bg_color"], camrotc2w=r["camrotc2w"], pixel_idx=r["pixel_idx"],
               near=r["near"], far=r["far"], h=r["h"], w=r["w"], intrinsic=r["intrinsic"])


@pytest.mark.parametrize("precision,bwd_fp32", [("bf16x3", 0), ("bf16x3", 1), ("bf16x3", 4), ("fp32", 0)])
@pytest.mark.parametrize("name", ["tiny_opaque", "tiny_thin_sr8", "tiny_order1", "tiny_raydist0_bg"])
def test_gradients_match_reference_fixture(name, precision, bwd_fp32, golden_dir):
    """bwd_fp32 = 0: every layer GEMM of the backward on the tensor cores (wgmma, BF16x3; default); 4: the forward recompute on the
    fp32 CUDA-core tiles (fp32-faithful LeakyReLU masks), dX / dW on the tensor cores; 1: everything on the fp32 tiles.  Modes 1 and 4
    meet the strict tolerance on every tensor; mode 0 on the MLP tensors and points_conf, and on all but a handful of points."""
    fx = golden.load(golden_dir, name)
    cfg = scene.CONFIGS["tiny"]
    order = int(fx["agg_intrp_order"]) if "agg_intrp_order" in fx.files else 2       # tiny_order1: the reference run with --agg_intrp_order 1
    # tiny_raydist0_bg: the reference run with --raydist_mode_unit 0 and bg_color (0.9, 0.1, 0.4)
    mode_unit = int(fx["raydist_mode_unit"]) if "raydist_mode_unit" in fx.files else 1
    bg = fx["bg_color"].tolist() if "bg_color" in fx.files else (1.0, 1.0, 1.0)
    net, pts, opt = harness.build_model(cfg, DEV, SR=int(fx["SR"]), max_o=100000, pnb_precision=precision, pnb_bwd_fp32=bwd_fp32, agg_intrp_order=order,
                                        raydist_mode_unit=mode_unit)
    net.aggregator.load_state_dict({k[4:]: torch.from_numpy(fx[k]) for k in fx.files if k.startswith("mlp.")})
    out = _forward(net, cfg, scene.make_rays(cfg, fx["pixels"], bg_color=bg))
    assert np.abs(out["coarse_raycolor"][0].detach().cpu().numpy() - fx["coarse_raycolor"]).max() <= 1e-4
    assert np.abs(out["weight"][0].cpu().numpy() - fx["weight"]).max() <= 1e-5
    assert np.abs(out["conf_coefficient"][0].detach().cpu().numpy() - fx["conf_coefficient"]).max() <= 1e-6
    assert np.abs(out["blend_weight"][0].cpu().numpy() - fx["blend_weight"]).max() <= 1e-4
    loss = (out["coarse_raycolor"] ** 2).sum() + 1e-3 * out["conf_coefficient"].sum()   # same loss as make_golden.py
    loss.backward()
    npn = net.neural_points
    per_point = _close_points if bwd_fp32 == 0 else _close
    per_point(npn.points_embeding.grad.cpu(), fx["grad_embedding"], "points_embeding")
    per_point(npn.points_color.grad.cpu(), fx["grad_color"], "points_color")
    per_point(npn.points_dir.grad.cpu(), fx["grad_dir"], "points_dir")
    _close(npn.points_conf.grad.cpu(), fx["grad_conf"], "points_conf", rtol=1e-3)
    for k, p in net.aggregator.named_parameters():     # (a flipped mask also moves one column of one weight gradient: 1e-3 for the tensor-core recompute)
        _close(p.grad.cpu(), fx["gradmlp." + k], "aggregator." + k, rtol=1e-3 if bwd_fp32 == 0 else 3e-4)
    assert npn.xyz.grad is None
    net.check_errors()


def test_gradients_match_oracle_autograd_chair():
    """BASELINE config 1 size (N=10k, 256 rays = 16x16 patch): backward against autograd through the oracle."""
    cfg = scene.CONFIGS["chair_plumbing"]
    net, pts, opt = harness.build_model(cfg, DEV, alpha_bias=3.0, seed=3)
    rays = scene.make_rays(cfg, scene.centre_patch(cfg, 16))
    out = _forward(net, cfg, rays)
    target = torch.linspace(0, 1, out["coarse_raycolor"].numel(), device=DEV).view_as(out["coarse_raycolor"])
    ((out["coarse_raycolor"] - target) ** 2).mean().backward()
    # oracle
    ref = pipeline.render(pts, harness.mlp_cpu(net.aggregator), rays["raydir"][0], cfg.campos, np.eye(3, dtype=np.float32),
                          cfg.near, cfg.far, opt.vsize, opt.vscale, opt.kernel_size, opt.query_size, opt.ranges, opt.SR,
                          opt.K, opt.P, pts["xyz"].shape[0], D=cfg.D, want_shade=False)
    pts_g = {k: v.clone().requires_grad_(k in ("embedding", "color", "dir", "conf")) for k, v in pts.items()}
    mlp_g = {k: v.clone().requires_grad_(True) for k, v in harness.mlp_cpu(net.aggregator).items()}
    mask = torch.from_numpy(ref["ray_mask"]) > 0
    sh = shade_oracle.shade(pts_g, mlp_g, torch.from_numpy(ref["sample_pidx"]), torch.from_numpy(ref["sample_loc_w"]),
                            rays["raydir"][0][mask], torch.tensor(cfg.campos), torch.eye(3), opt.vsize, torch.ones(3))
    ((sh["ray_color"][None] - target.cpu()) ** 2).mean().backward()
    npn = net.neural_points
    _close(npn.points_embeding.grad.cpu(), pts_g["embedding"].grad, "points_embeding")
    _close(npn.points_color.grad.cpu(), pts_g["color"].grad, "points_color")
    _close(npn.points_dir.grad.cpu(), pts_g["dir"].grad, "points_dir")
    _close(npn.points_conf.grad.cpu(), pts_g["conf"].grad, "points_conf", rtol=1e-3)
    for k, p in net.aggregator.named_parameters():
        _close(p.grad.cpu(), mlp_g[k].grad, "aggregator." + k)


def test_optimisation_step_reduces_loss():
    """A few Adam steps on the point features + MLP through the CUDA backward lower an image loss (end-to-end sanity
    of forward + backward + in-place parameter updates + weight re-packing)."""
    cfg = scene.CONFIGS["tiny"]
    net, pts, opt = harness.build_model(cfg, DEV, alpha_bias=4.0)
    rays = scene.make_rays(cfg, scene.centre_patch(cfg, 32))
    params = [p for p in net.parameters() if p.requires_grad]
    optim = torch.optim.Adam(params, lr=2e-3)
    losses = []
    for it in range(6):
        optim.zero_grad()
        out = _forward(net, cfg, rays)
        loss = ((out["coarse_raycolor"] - 0.25) ** 2).mean()
        loss.backward()
        optim.step()
        losses.append(float(loss.detach()))
    assert losses[-1] < losses[0] * 0.9, losses


def test_gradients_with_jittered_t_table():
    """Training marches a per-ray jittered t table (point_query.py:81): same explicit table to the CUDA path and to the oracle."""
    from pointnerf_b200.point_query import device_t_table_jitter
    cfg = scene.CONFIGS["chair_plumbing"]
    net, pts, opt = harness.build_model(cfg, DEV, alpha_bias=3.0, seed=5)
    rays = scene.make_rays(cfg, scene.centre_patch(cfg, 16))
    R = rays["raydir"].shape[1]
    g = torch.Generator(device=DEV).manual_seed(9)
    t = device_t_table_jitter(cfg.near, cfg.far, cfg.D, R, 0.3, torch.device(DEV), generator=g)
    net.neural_points.querier._t_for = lambda near, far, n, device: t          # what is_train draws internally, made explicit
    out = _forward(net, cfg, rays)
    target = torch.linspace(0, 1, out["coarse_raycolor"].numel(), device=DEV).view_as(out["coarse_raycolor"])
    ((out["coarse_raycolor"] - target) ** 2).mean().backward()
    ref = pipeline.render(pts, harness.mlp_cpu(net.aggregator), rays["raydir"][0], cfg.campos, np.eye(3, dtype=np.float32),
                          cfg.near, cfg.far, opt.vsize, opt.vscale, opt.kernel_size, opt.query_size, opt.ranges, opt.SR,
                          opt.K, opt.P, pts["xyz"].shape[0], D=cfg.D, t=t.cpu().numpy(), want_shade=False)
    assert np.array_equal(out["ray_mask"][0].cpu().numpy(), ref["ray_mask"])
    pts_g = {k: v.clone().requires_grad_(k in ("embedding", "color", "dir", "conf")) for k, v in pts.items()}
    mlp_g = {k: v.clone().requires_grad_(True) for k, v in harness.mlp_cpu(net.aggregator).items()}
    mask = torch.from_numpy(ref["ray_mask"]) > 0
    sh = shade_oracle.shade(pts_g, mlp_g, torch.from_numpy(ref["sample_pidx"]), torch.from_numpy(ref["sample_loc_w"]),
                            rays["raydir"][0][mask], torch.tensor(cfg.campos), torch.eye(3), opt.vsize, torch.ones(3))
    assert (out["coarse_raycolor"][0].detach().cpu() - sh["ray_color"]).abs().max().item() <= 1e-4
    ((sh["ray_color"][None] - target.cpu()) ** 2).mean().backward()
    npn = net.neural_points
    _close(npn.points_embeding.grad.cpu(), pts_g["embedding"].grad, "points_embeding")
    _close(npn.points_color.grad.cpu(), pts_g["color"].grad, "points_color")
    _close(npn.points_dir.grad.cpu(), pts_g["dir"].grad, "points_dir")
    _close(npn.points_conf.grad.cpu(), pts_g["conf"].grad, "points_conf", rtol=1e-3)
    for k, p in net.aggregator.named_parameters():
        _close(p.grad.cpu(), mlp_g[k].grad, "aggregator." + k)


def test_backward_of_an_overwritten_forward_is_refused():
    """The backward recomputes from the module's query / sigma_rgb buffers: a second forward (or an eval render) before backward()
    would silently change them -> PnbError instead of wrong gradients."""
    from pointnerf_b200.lib import PnbError
    cfg = scene.CONFIGS["tiny"]
    net, pts, opt = harness.build_model(cfg, DEV, alpha_bias=4.0)
    rays = scene.make_rays(cfg, scene.centre_patch(cfg, 24))
    out1 = _forward(net, cfg, rays)
    with torch.no_grad():
        _forward(net, cfg, scene.make_rays(cfg, scene.centre_patch(cfg, 12)))      # e.g. a validation render in between
    with pytest.raises(PnbError):
        (out1["coarse_raycolor"] ** 2).sum().backward()
    out2 = _forward(net, cfg, rays)
    (out2["coarse_raycolor"] ** 2).sum().backward()                                   # the normal order works
    assert net.neural_points.points_embeding.grad is not None
