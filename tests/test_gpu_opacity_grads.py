"""GPU: gradients of losses on coarse_is_background and coarse_point_opacity (the reference's bg_loss and zero_one terms,
base_rendering_model.py:620-641) through the fused backward: against the reference's own autograd (tests/golden/tiny_opacity_loss,
oracle/make_golden_opacity.py), against autograd through the oracle on other configurations, and against the colour-only backward,
which a loss that adds these outputs with weight zero must reproduce."""
import numpy as np
import pytest
import torch
import torch.nn.functional as F

from oracle import golden, pipeline, shade_oracle_rw2c
from oracle.make_golden_opacity import CASES, fill_rays, gt_mask_of, opacity_loss
from pointnerf_b200 import harness, scene

pytestmark = pytest.mark.gpu
DEV = "cuda:0"


def _close(a, ref, name, rtol=3e-4):
    a, ref = np.asarray(a, np.float64), np.asarray(ref, np.float64).reshape(np.asarray(a).shape)
    scale = max(np.abs(ref).max(), 1e-6)
    d = np.abs(a - ref).max()
    assert d <= rtol * scale + 1e-7, "%s: max abs diff %.3e vs scale %.3e" % (name, d, scale)


def _close_points(a, ref, name, rtol=3e-4, max_outlier_frac=0.01, outlier_rtol=2e-2):
    """The tolerance of tests/test_gpu_backward.py for the tensor-core recompute: strict on all but <= 1 % of the points (those whose
    pair crossed a LeakyReLU mask flip of the BF16x3 recompute), bounded on those."""
    a, ref = np.asarray(a, np.float64)[0], np.asarray(ref, np.float64).reshape(np.asarray(a).shape)[0]
    scale = max(np.abs(ref).max(), 1e-6)
    d = np.abs(a - ref).max(axis=-1)
    bad = d > rtol * scale + 1e-7
    assert bad.sum() <= max(4, max_outlier_frac * d.shape[0]), "%s: %d of %d points beyond %.0e of scale" % (name, int(bad.sum()), d.shape[0], rtol)
    assert d.max() <= outlier_rtol * scale, "%s: max abs diff %.3e vs scale %.3e" % (name, d.max(), scale)


def _forward(net, rays):
    r = {k: v.to(DEV) for k, v in rays.items()}
    return net(r["campos"], r["raydir"], bg_color=r["bg_color"], camrotc2w=r["camrotc2w"], pixel_idx=r["pixel_idx"],
               near=r["near"], far=r["far"], h=r["h"], w=r["w"], intrinsic=r["intrinsic"])


def _loss_of(out, gt_mask, **weights):
    """opacity_loss on the module's outputs, with coarse_is_background / coarse_point_opacity filled to every ray as fill_invalid does."""
    hit = out["ray_mask"][0]
    return opacity_loss(out["coarse_raycolor"][0], out["conf_coefficient"], fill_rays(hit, out["coarse_is_background"][0], 1.0),
                        fill_rays(hit, out["coarse_point_opacity"][0], 0.0), gt_mask.to(DEV), **weights)


def _check_grads(net, ref_points, ref_mlp, bwd_fp32):
    """ref_points: name -> reference gradient of the 4 point tensors; ref_mlp: aggregator parameter name -> gradient (None: the loss
    does not reach that tensor, whose gradient must then be zero)."""
    npn = net.neural_points
    per_point = _close_points if bwd_fp32 == 0 else _close
    for k in ("points_embeding", "points_color", "points_dir"):
        per_point(getattr(npn, k).grad.cpu(), ref_points[k], k)
    _close(npn.points_conf.grad.cpu(), ref_points["points_conf"], "points_conf", rtol=1e-3)
    for k, p in net.aggregator.named_parameters():
        ref = ref_mlp[k]
        if ref is None:
            assert torch.count_nonzero(p.grad).item() == 0, k
        else:
            _close(p.grad.cpu(), ref, "aggregator." + k, rtol=1e-3 if bwd_fp32 == 0 else 3e-4)
    assert npn.xyz.grad is None
    net.check_errors()


@pytest.mark.parametrize("precision,bwd_fp32", [(p, b) for p in ("bf16x3", "fp32") for b in (0, 1, 4)])
@pytest.mark.parametrize("name", [c[0] for c in CASES])
def test_gradients_match_reference_fixture(name, precision, bwd_fp32, golden_dir):
    fx = golden.load(golden_dir, name)
    gx = golden.load(golden_dir, "tiny_opacity_loss")
    cfg = scene.CONFIGS["tiny"]
    net, pts, opt = harness.build_model(cfg, DEV, SR=int(fx["SR"]), max_o=100000, pnb_precision=precision, pnb_bwd_fp32=bwd_fp32)
    net.aggregator.load_state_dict({k[4:]: torch.from_numpy(fx[k]) for k in fx.files if k.startswith("mlp.")})
    out = _forward(net, scene.make_rays(cfg, fx["pixels"]))
    assert np.array_equal(out["ray_mask"][0].cpu().numpy(), fx["ray_mask"])
    loss = _loss_of(out, torch.from_numpy(gx[name + ".gt_mask"]), bg_weight=float(gx["bg_weight"]),
                    zero_one_weight=float(gx["zero_one_weight"]))
    assert abs(loss.item() - float(gx[name + ".loss"])) <= 1e-4 * abs(float(gx[name + ".loss"]))
    loss.backward()
    _check_grads(net, {k: gx[name + ".grad_" + s] for k, s in (("points_embeding", "embedding"), ("points_color", "color"),
                                                              ("points_dir", "dir"), ("points_conf", "conf"))},
                 {k: gx[name + ".gradmlp." + k] for k, _ in net.aggregator.named_parameters()}, bwd_fp32)


def _oracle_grads(cfg, opt, pts, agg, rays, R, loss_fn):
    """Autograd through the oracle (query: oracle/pipeline.py; shading: oracle/shade_oracle_rw2c.py, which hands a [3,3] frame to
    oracle/shade_oracle.py) of loss_fn(shade outputs, hit-ray mask)."""
    raydir = rays["raydir"][0]
    ref = pipeline.render(pts, harness.mlp_cpu(agg), raydir, cfg.campos, np.eye(3, dtype=np.float32), cfg.near, cfg.far,
                          opt.vsize, opt.vscale, opt.kernel_size, opt.query_size, opt.ranges, opt.SR, opt.K, opt.P,
                          opt.max_o if opt.max_o is not None else pts["xyz"].shape[0], D=cfg.D, want_shade=False)
    hit = torch.from_numpy(ref["ray_mask"])
    pts_g = {k: v.clone().requires_grad_(k in ("embedding", "color", "dir", "conf")) for k, v in pts.items()}
    pts_g["Rw2c"] = R
    mlp_g = {k: v.clone().requires_grad_(True) for k, v in harness.mlp_cpu(agg).items()}
    sh = shade_oracle_rw2c.shade(pts_g, mlp_g, torch.from_numpy(ref["sample_pidx"]), torch.from_numpy(ref["sample_loc_w"]),
                                 raydir[hit > 0], torch.tensor(cfg.campos), torch.eye(3), opt.vsize, torch.ones(3),
                                 agg_intrp_order=opt.agg_intrp_order)
    loss_fn(sh, hit).backward()
    points = {"points_" + k: pts_g[s].grad for k, s in (("embeding", "embedding"), ("color", "color"), ("dir", "dir"), ("conf", "conf"))}
    return hit, points, {k: v.grad for k, v in mlp_g.items()}


def test_background_loss_alone_matches_oracle_autograd_chair():
    """A loss made of the bg_loss term alone (no colour, no conf term): the backward has no colour gradient (d_ray_color NULL), and the
    colour branch, which bg_T does not depend on, receives exactly zero."""
    cfg = scene.CONFIGS["chair_plumbing"]
    net, pts, opt = harness.build_model(cfg, DEV, alpha_bias=3.0, seed=3)
    rays = scene.make_rays(cfg, scene.centre_patch(cfg, 16))
    gt_mask = gt_mask_of(rays["raydir"].shape[1], seed=1)

    def bg_loss(is_background, hit):
        return F.mse_loss(fill_rays(hit, is_background, 1.0) * (1 - gt_mask.to(is_background.device)),
                          1 - gt_mask.to(is_background.device))

    out = _forward(net, rays)
    bg_loss(out["coarse_is_background"][0], out["ray_mask"][0]).backward()
    hit, ref_points, ref_mlp = _oracle_grads(cfg, opt, pts, net.aggregator, rays, torch.eye(3), lambda sh, h: bg_loss(sh["bg_T"], h))
    assert np.array_equal(out["ray_mask"][0].cpu().numpy(), hit.numpy())
    for k, p in net.aggregator.named_parameters():
        if k.startswith("color_branch"):
            assert ref_mlp[k] is None or torch.count_nonzero(ref_mlp[k]).item() == 0, k
            assert torch.count_nonzero(p.grad).item() == 0, k
    _check_grads(net, ref_points, ref_mlp, 0)


@pytest.mark.parametrize("case", ["order1", "per_point_frames"])
def test_gradients_match_oracle_autograd(case):
    """agg_intrp_order 1 (alpha_branch on the K-aggregated feature) and an edited scene with per-point frames (scene.edit_frames)."""
    cfg = scene.CONFIGS["tiny"]
    over = dict(agg_intrp_order=1) if case == "order1" else {}
    net, pts, opt = harness.build_model(cfg, DEV, alpha_bias=4.0, **over)
    R = torch.eye(3)
    if case == "per_point_frames":
        R = scene.edit_frames(pts["xyz"])
        p = net.neural_points
        p.set_points(p.xyz.detach().clone(), p.points_embeding.detach().clone(), points_color=p.points_color.detach().clone(),
                     points_dir=p.points_dir.detach().clone(), points_conf=p.points_conf.detach().clone(), Rw2c=R.to(DEV))
    rays = scene.make_rays(cfg, scene.centre_patch(cfg, 32))
    gt_mask = gt_mask_of(rays["raydir"].shape[1])
    out = _forward(net, rays)
    _loss_of(out, gt_mask).backward()
    hit, ref_points, ref_mlp = _oracle_grads(
        cfg, opt, pts, net.aggregator, rays, R,
        lambda sh, h: opacity_loss(sh["ray_color"], sh["conf_coefficient"], fill_rays(h, sh["bg_T"], 1.0), fill_rays(h, sh["opacity"], 0.0), gt_mask))
    assert np.array_equal(out["ray_mask"][0].cpu().numpy(), hit.numpy())
    _check_grads(net, ref_points, ref_mlp, 0)


# weight gradients the tensor-core backward reduces with its deterministic split-K (csrc/backward.cu, gemm_tn_acc); the biases (colsum),
# the alpha branch, colour_branch.6 and the point gradients are accumulated with atomics, whose order varies from run to run
DETERMINISTIC_GRADS = tuple("aggregator.%s.weight" % k for k in
                            ("block1.0", "block1.2", "block3.0", "block3.2", "color_branch.0", "color_branch.2", "color_branch.4"))


def test_zero_weight_terms_give_the_colour_loss_gradients():
    """Adding opacity and bg_T to a colour loss with weight zero takes the kernel path with upstream opacity / bg_T gradients, which then
    reads zeros; it must reduce to the colour-only path: the same gradients, bitwise wherever the backward reduces deterministically,
    and within the run-to-run spread of its atomics elsewhere."""
    cfg = scene.CONFIGS["tiny"]
    net, pts, opt = harness.build_model(cfg, DEV, alpha_bias=4.0)
    rays = scene.make_rays(cfg, scene.centre_patch(cfg, 48))

    def step(zero_terms):
        for p in net.parameters():
            p.grad = None
        out = _forward(net, rays)
        loss = (out["coarse_raycolor"] ** 2).sum() + 1e-3 * out["conf_coefficient"].sum()
        if zero_terms:
            loss = loss + 0 * (out["coarse_point_opacity"].sum() + out["coarse_is_background"].sum())
        loss.backward()
        return {k: p.grad.detach().clone() for k, p in net.named_parameters() if p.grad is not None}

    g_col, g_zero = step(False), step(True)
    assert set(g_col) == set(g_zero) and set(DETERMINISTIC_GRADS) <= set(g_col)
    for k in g_col:
        if k in DETERMINISTIC_GRADS:
            assert torch.equal(g_col[k], g_zero[k]), k
        else:
            _close(g_zero[k].cpu(), g_col[k].cpu(), k, rtol=1e-5)
    net.check_errors()


def test_conf_coefficient_loss_alone_does_not_reach_the_shading_backward():
    """A training loss on conf_coefficient alone (the harness default zero_one_loss_items, or a separate backward of such a term):
    points_conf gets the straight-through gradient of the clamp, equal to the oracle's, and nothing else gets a gradient - the
    blend_weight kernel's opacity input carries no graph, so the shading backward is not run."""
    cfg = scene.CONFIGS["tiny"]
    net, pts, opt = harness.build_model(cfg, DEV, alpha_bias=4.0)
    rays = scene.make_rays(cfg, scene.centre_patch(cfg, 32))
    out = _forward(net, rays)
    out["conf_coefficient"].sum().backward()
    hit, ref_points, _ = _oracle_grads(cfg, opt, pts, net.aggregator, rays, torch.eye(3), lambda sh, h: sh["conf_coefficient"].sum())
    assert np.array_equal(out["ray_mask"][0].cpu().numpy(), hit.numpy())
    npn = net.neural_points
    assert torch.equal(npn.points_conf.grad.cpu(), ref_points["points_conf"])
    assert npn.points_embeding.grad is None and npn.points_color.grad is None and npn.points_dir.grad is None
    assert all(p.grad is None for p in net.aggregator.parameters())
    net.check_errors()


def test_training_outputs_that_require_grad():
    """As in the reference: coarse_point_opacity and coarse_is_background stay in the graph; weight and blend_weight are detached
    (neural_points_volumetric_model.py:325-327), and ray_mask is an integer mask."""
    cfg = scene.CONFIGS["tiny"]
    net, pts, opt = harness.build_model(cfg, DEV, alpha_bias=4.0)
    out = _forward(net, scene.make_rays(cfg, scene.centre_patch(cfg, 16)))
    for k in ("coarse_raycolor", "coarse_point_opacity", "coarse_is_background", "conf_coefficient"):
        assert out[k].requires_grad, k
    for k in ("weight", "blend_weight", "ray_mask"):
        assert not out[k].requires_grad, k
    with torch.no_grad():
        out = _forward(net, scene.make_rays(cfg, scene.centre_patch(cfg, 16)))
    assert not any(v.requires_grad for v in out.values())
