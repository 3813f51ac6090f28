"""GPU: the DTU configuration, point_features_dim 63 with point_{conf,dir,color}_mode "01", through the fused path (the F = 63
instantiations of k_point_pre, k_shade_wg, k_shade_fwd, k_bwd_build and k_bwd_scatter).  Forward and gradients against the
reference-generated fixtures tests/golden/tiny_feat63 (agg_intrp_order 2) and tiny_feat63_order1, per-point frames and other
configurations against the oracle (oracle/shade_oracle.py, generic in the width), and the whole-image entry point."""
import numpy as np
import pytest
import torch

from oracle import golden, pipeline, shade_oracle_rw2c
from pointnerf_b200 import harness, lib, runner, scene

pytestmark = pytest.mark.gpu
DEV = "cuda:0"
TOL = 1e-4
PRECISIONS = ["bf16x3", "bf16x3-general", "fp32"]
CASES = ["tiny_feat63", "tiny_feat63_order1"]


def _prec(precision):
    """bf16x3: the frozen-cloud pair kernel for renders; bf16x3-general: the general pair kernel; fp32: the CUDA-core kernel."""
    if precision == "bf16x3-general":
        return dict(pnb_precision="bf16x3", pnb_frozen=0)
    return dict(pnb_precision=precision)


def _forward(net, rays):
    r = {k: v.to(DEV) for k, v in rays.items()}
    return net(r["campos"], r["raydir"], bg_color=r["bg_color"], camrotc2w=r["camrotc2w"], pixel_idx=r["pixel_idx"],
               near=r["near"], far=r["far"], h=r["h"], w=r["w"], intrinsic=r["intrinsic"])


def _render_full(net, cfg, rays):
    with torch.no_grad():
        return net.render_full(list(cfg.campos), rays["raydir"].to(DEV), torch.eye(3), cfg.near, cfg.far, [1., 1., 1.])


def _fixture_net(fx, **over):
    cfg = scene.CONFIGS["tiny"]
    net, pts, opt = harness.build_model(cfg, DEV, SR=int(fx["SR"]), max_o=100000, feat_dim=63,
                                        agg_intrp_order=int(fx["agg_intrp_order"]), **over)
    net.aggregator.load_state_dict({k[4:]: torch.from_numpy(fx[k]) for k in fx.files if k.startswith("mlp.")})
    assert np.array_equal(net.neural_points.points_embeding.detach().cpu().numpy(), fx["embedding63"])
    return cfg, net


def _oracle_render(cfg, opt, net, raydir, R=None):
    """The oracle pipeline (query) with the shading restatement on the module's own 63-channel points."""
    npn = net.neural_points
    pts = dict(xyz=npn.xyz.detach().cpu(), embedding=npn.points_embeding.detach().cpu(), color=npn.points_color.detach().cpu(),
               dir=npn.points_dir.detach().cpu(), conf=npn.points_conf.detach().cpu(), Rw2c=torch.eye(3) if R is None else R)
    ref = pipeline.render(pts, harness.mlp_cpu(net.aggregator), raydir, cfg.campos, np.eye(3, dtype=np.float32), cfg.near, cfg.far,
                          opt.vsize, opt.vscale, opt.kernel_size, opt.query_size, opt.ranges, opt.SR, opt.K, opt.P,
                          opt.max_o if opt.max_o is not None else pts["xyz"].shape[0], D=cfg.D, want_shade=False)
    mask = torch.from_numpy(ref["ray_mask"]) > 0
    assert int(mask.sum()) > 0
    sh = shade_oracle_rw2c.shade(pts, harness.mlp_cpu(net.aggregator), torch.from_numpy(ref["sample_pidx"]),
                                 torch.from_numpy(ref["sample_loc_w"]), raydir[mask], torch.tensor(cfg.campos), torch.eye(3), opt.vsize,
                                 torch.ones(3), agg_intrp_order=opt.agg_intrp_order)
    ref.update(sh)
    ref.update(shade_oracle_rw2c.fill_invalid(mask, sh["ray_color"], sh["opacity"], sh["bg_T"], sh["queried_shading"], torch.ones(3)))
    return ref


def _close(a, ref, name, rtol=3e-4):
    a, ref = np.asarray(a, np.float64), np.asarray(ref, np.float64).reshape(np.asarray(a).shape)
    scale = max(np.abs(ref).max(), 1e-6)
    d = np.abs(a - ref).max()
    assert d <= rtol * scale + 1e-7, "%s: max abs diff %.3e vs scale %.3e" % (name, d, scale)


def _close_points(a, ref, name, rtol=3e-4, max_outlier_frac=0.01, outlier_rtol=2e-2):
    """The tolerance of tests/test_gpu_rw2c.py for the tensor-core recompute: strict on all but <= 1 % of the points (those whose pair
    crossed a LeakyReLU mask flip of the BF16x3 recompute), bounded on those."""
    a, ref = np.asarray(a, np.float64)[0], np.asarray(ref, np.float64).reshape(np.asarray(a).shape)[0]
    scale = max(np.abs(ref).max(), 1e-6)
    d = np.abs(a - ref).max(axis=-1)
    bad = d > rtol * scale + 1e-7
    assert bad.sum() <= max(4, max_outlier_frac * d.shape[0]), "%s: %d of %d points beyond %.0e of scale" % (name, int(bad.sum()), d.shape[0], rtol)
    assert d.max() <= outlier_rtol * scale, "%s: max abs diff %.3e vs scale %.3e" % (name, d.max(), scale)


@pytest.mark.parametrize("name", CASES)
@pytest.mark.parametrize("precision", PRECISIONS)
def test_forward_matches_reference_fixture(golden_dir, precision, name):
    fx = golden.load(golden_dir, name)
    cfg, net = _fixture_net(fx, **_prec(precision))
    with torch.no_grad():
        out = _forward(net, scene.make_rays(cfg, fx["pixels"]))
    assert np.array_equal(out["ray_mask"][0].cpu().numpy(), fx["ray_mask"])
    for k in ("coarse_raycolor", "coarse_point_opacity", "coarse_is_background"):
        d = np.abs(out[k][0].cpu().numpy() - fx[k]).max()
        assert d <= TOL, "%s max abs diff %.3e" % (k, d)
    net.check_errors()


@pytest.mark.parametrize("name", CASES)
@pytest.mark.parametrize("precision,bwd_fp32", [("bf16x3", 0), ("bf16x3", 1), ("bf16x3", 4), ("fp32", 0)])
def test_gradients_match_reference_fixture(golden_dir, precision, bwd_fp32, name):
    fx = golden.load(golden_dir, name)
    cfg, net = _fixture_net(fx, pnb_precision=precision, pnb_bwd_fp32=bwd_fp32)
    out = _forward(net, scene.make_rays(cfg, fx["pixels"]))
    assert np.abs(out["coarse_raycolor"][0].detach().cpu().numpy() - fx["coarse_raycolor"]).max() <= TOL
    loss = (out["coarse_raycolor"] ** 2).sum() + 1e-3 * out["conf_coefficient"].sum()   # the loss of oracle/make_golden_feat63.py
    loss.backward()
    npn = net.neural_points
    assert npn.points_embeding.grad.shape == (1, cfg.N, 63)
    # the point gradients take the bounded-outlier comparison in every backward mode: with 501 inputs, the fp32 block1.0 pre-activations
    # of a few pairs also round to the other side of zero than the reference's (another summation order), and each such LeakyReLU mask
    # flip moves that pair's point gradients by up to ~1e-3 of scale
    _close_points(npn.points_embeding.grad.cpu(), fx["grad_embedding"], "points_embeding")
    _close_points(npn.points_color.grad.cpu(), fx["grad_color"], "points_color")
    _close_points(npn.points_dir.grad.cpu(), fx["grad_dir"], "points_dir")
    _close(npn.points_conf.grad.cpu(), fx["grad_conf"], "points_conf", rtol=1e-3)
    for k, p in net.aggregator.named_parameters():
        _close(p.grad.cpu(), fx["gradmlp." + k], "aggregator." + k, rtol=1e-3 if bwd_fp32 == 0 else 3e-4)
    assert npn.xyz.grad is None
    net.check_errors()


@pytest.mark.parametrize("order", [2, 1])
@pytest.mark.parametrize("precision", PRECISIONS)
def test_per_point_frames_at_63_channels(precision, order):
    """Per-point frames (Rw2c [N,3,3], two objects) combine with the width: a chunk against the oracle."""
    cfg = scene.CONFIGS["tiny"]
    net, pts, opt = harness.build_model(cfg, DEV, alpha_bias=4.0, feat_dim=63, agg_intrp_order=order, **_prec(precision))
    R = scene.edit_frames(pts["xyz"])
    net.neural_points.Rw2c = torch.nn.Parameter(R.to(DEV), requires_grad=False)
    rays = scene.make_rays(cfg, scene.centre_patch(cfg, 64))
    out = _render_full(net, cfg, rays)
    ref = _oracle_render(cfg, opt, net, rays["raydir"][0], R)
    assert np.array_equal(out["ray_mask"][0].cpu().numpy(), ref["ray_mask"])
    for a in ("coarse_raycolor", "coarse_point_opacity", "coarse_is_background"):
        d = (out[a][0].cpu() - ref[a]).abs().max().item()
        assert d <= TOL, "%s max abs diff %.3e" % (a, d)
    net.check_errors()


@pytest.mark.parametrize("precision", PRECISIONS)
def test_render_image_63_channels(precision):
    """runner.render_image on a 63-channel cloud: the whole tiny frame against the oracle, and bit for bit the reference's chunk loop
    (runner.render_image_chunked)."""
    cfg = scene.CONFIGS["tiny"]
    net, pts, opt = harness.build_model(cfg, DEV, alpha_bias=3.0, feat_dim=63, **_prec(precision))
    px, py = np.meshgrid(np.arange(cfg.W), np.arange(cfg.H))
    rays = scene.make_rays(cfg, np.stack((px, py), -1).reshape(-1, 2).astype(np.float32))
    data = {k: (v.to(DEV) if isinstance(v, torch.Tensor) else v) for k, v in rays.items()}
    whole = runner.render_image(net, data, cfg.H, cfg.W)
    chunked = runner.render_image_chunked(net, data, cfg.H, cfg.W, 1024)
    assert np.array_equal(whole["coarse_raycolor"].cpu().numpy(), chunked["coarse_raycolor"])
    ref = _oracle_render(cfg, opt, net, rays["raydir"][0])
    assert np.array_equal(whole["ray_mask"].reshape(-1).cpu().numpy(), ref["ray_mask"])
    d = (whole["coarse_raycolor"].reshape(-1, 3).cpu() - ref["coarse_raycolor"]).abs().max().item()
    assert d <= TOL, "coarse_raycolor max abs diff %.3e" % d
    net.check_errors()


def test_install_into_reference_shaped_module_63_channels():
    """Seam B (INTEGRATION.md) with a DTU-shaped module: points_embeding [1,N,63] beside colour / dir / conf, block1.0 [256, 501]."""
    import torch.nn as nn
    from pointnerf_b200 import ray_marching as P
    from pointnerf_b200.point_query import lighting_fast_querier

    cfg = scene.CONFIGS["tiny"]
    opt = harness.make_opt(cfg, feat_dim=63)
    ours, pts, _ = harness.build_model(cfg, DEV, alpha_bias=4.0, feat_dim=63)
    src = ours.neural_points

    class RefNeuralPoints(nn.Module):
        def __init__(self):
            super().__init__()
            self.opt = opt
            self.xyz = nn.Parameter(src.xyz.detach().clone(), requires_grad=False)
            self.points_embeding = nn.Parameter(src.points_embeding.detach().clone())
            self.points_conf = nn.Parameter(src.points_conf.detach().clone())
            self.points_dir = nn.Parameter(src.points_dir.detach().clone())
            self.points_color = nn.Parameter(src.points_color.detach().clone())
            self.Rw2c = torch.eye(3, device=DEV)
            self.querier = lighting_fast_querier(torch.device(DEV), opt)

    class RefRayMarching(nn.Module):
        def __init__(self, aggregator, neural_points, opt):
            super().__init__()
            self.aggregator, self.neural_points, self.opt = aggregator, neural_points, opt

        def forward(self, *a, **k):
            raise AssertionError("the eager reference forward must have been replaced")

    P.install_into(RefRayMarching)
    net = RefRayMarching(ours.aggregator, RefNeuralPoints(), opt)
    rays = scene.make_rays(cfg, scene.centre_patch(cfg, 32))
    with torch.no_grad():
        out = _forward(net, rays)
    ref = _oracle_render(cfg, opt, ours, rays["raydir"][0])
    assert np.array_equal(out["ray_mask"][0].cpu().numpy(), ref["ray_mask"])
    assert (out["coarse_raycolor"][0].cpu() - ref["ray_color"]).abs().max().item() <= TOL


def test_mismatched_widths_are_refused():
    """The C ABI checks that the MLP matches the points' width, and refuses widths without kernels."""
    cfg = scene.CONFIGS["tiny"]
    net, pts, opt = harness.build_model(cfg, DEV, alpha_bias=4.0, feat_dim=63)
    l = lib.load()
    npn = net.neural_points
    desc = net._mlp.get(net.aggregator)
    p = npn.points_desc()
    assert p.feat_dim == 63 and desc.feat_dim == 63
    assert l.pnb_mlp_pack_bytes(63) > l.pnb_mlp_pack_bytes(32) == l.pnb_mlp_pack_bytes(0)
    assert l.pnb_mlp_pack_bytes(48) == 0 and l.pnb_backward_bytes(10, 100, 48) == 0
    assert l.pnb_backward_bytes(10, 100, 63) > l.pnb_backward_bytes(10, 100, 32)
    pre = torch.empty(cfg.N * 256, device=DEV)
    stream = torch.cuda.current_stream().cuda_stream
    p.feat_dim = 32
    assert l.pnb_point_pre(lib.C.byref(p), lib.C.byref(desc), pre.data_ptr(), pre.numel() * 4, stream) == -1
    assert b"point_features_dim" in l.pnb_last_error()
    p.feat_dim = 48
    assert l.pnb_point_pre(lib.C.byref(p), lib.C.byref(desc), pre.data_ptr(), pre.numel() * 4, stream) == -4
    torch.cuda.synchronize()
