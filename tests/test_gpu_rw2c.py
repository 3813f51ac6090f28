"""GPU: per-point world->canonical rotations (neural_points.Rw2c [N,3,3], edited / composed scenes) through the fused path.
Forward and gradients against the reference-generated fixture tests/golden/tiny_rw2c, the oracle (oracle/shade_oracle_rw2c.py) on
other configurations, and the uniform path: a per-point tensor whose rows all equal M must give what Rw2c = M gives, bit for bit."""
import numpy as np
import pytest
import torch

from oracle import golden, pipeline, shade_oracle_rw2c
from pointnerf_b200 import harness, scene
from pointnerf_b200.lib import PnbError

pytestmark = pytest.mark.gpu
DEV = "cuda:0"
TOL = 1e-4
PRECISIONS = ["bf16x3", "bf16x3-general", "fp32"]


def _prec(precision):
    """bf16x3: the frozen-cloud pair kernel for renders; bf16x3-general: the general pair kernel; fp32: the CUDA-core kernel."""
    if precision == "bf16x3-general":
        return dict(pnb_precision="bf16x3", pnb_frozen=0)
    return dict(pnb_precision=precision)


def _set_frames(net, R):
    """Re-installs the module's points with the frames R ([3,3] or [N,3,3]), as a loaded checkpoint would."""
    p = net.neural_points
    p.set_points(p.xyz.detach().clone(), p.points_embeding.detach().clone(), points_color=p.points_color.detach().clone(),
                 points_dir=p.points_dir.detach().clone(), points_conf=p.points_conf.detach().clone(), Rw2c=R.to(DEV))


def _forward(net, rays):
    r = {k: v.to(DEV) for k, v in rays.items()}
    return net(r["campos"], r["raydir"], bg_color=r["bg_color"], camrotc2w=r["camrotc2w"], pixel_idx=r["pixel_idx"],
               near=r["near"], far=r["far"], h=r["h"], w=r["w"], intrinsic=r["intrinsic"])


def _render_full(net, cfg, rays):
    with torch.no_grad():
        return net.render_full(list(cfg.campos), rays["raydir"].to(DEV), torch.eye(3), cfg.near, cfg.far, [1., 1., 1.])


def _oracle_render(cfg, opt, pts, agg, raydir, R):
    """The oracle pipeline (oracle/pipeline.py: query) with the per-point shading restatement (oracle/shade_oracle_rw2c.py)."""
    ref = pipeline.render(pts, harness.mlp_cpu(agg), raydir, cfg.campos, np.eye(3, dtype=np.float32), cfg.near, cfg.far,
                          opt.vsize, opt.vscale, opt.kernel_size, opt.query_size, opt.ranges, opt.SR, opt.K, opt.P,
                          opt.max_o if opt.max_o is not None else pts["xyz"].shape[0], D=cfg.D, want_shade=False)
    mask = torch.from_numpy(ref["ray_mask"]) > 0
    assert int(mask.sum()) > 0
    pts = dict(pts)
    pts["Rw2c"] = R
    sh = shade_oracle_rw2c.shade(pts, harness.mlp_cpu(agg), torch.from_numpy(ref["sample_pidx"]), torch.from_numpy(ref["sample_loc_w"]),
                                 raydir[mask], torch.tensor(cfg.campos), torch.eye(3), opt.vsize, torch.ones(3),
                                 agg_intrp_order=opt.agg_intrp_order)
    ref.update(sh)
    ref.update(shade_oracle_rw2c.fill_invalid(mask, sh["ray_color"], sh["opacity"], sh["bg_T"], sh["queried_shading"], torch.ones(3)))
    return ref


def _fixture_net(fx, **over):
    cfg = scene.CONFIGS["tiny"]
    net, pts, opt = harness.build_model(cfg, DEV, SR=int(fx["SR"]), max_o=100000, **over)
    net.aggregator.load_state_dict({k[4:]: torch.from_numpy(fx[k]) for k in fx.files if k.startswith("mlp.")})
    _set_frames(net, torch.from_numpy(fx["Rw2c"]))
    return cfg, net


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


@pytest.mark.parametrize("precision", PRECISIONS)
def test_forward_matches_reference_fixture(golden_dir, precision):
    fx = golden.load(golden_dir, "tiny_rw2c")
    cfg, net = _fixture_net(fx, **_prec(precision))
    with torch.no_grad():
        out = _forward(net, scene.make_rays(cfg, fx["pixels"]))
    assert np.array_equal(out["ray_mask"][0].cpu().numpy(), fx["ray_mask"])
    for k in ("coarse_raycolor", "coarse_point_opacity", "coarse_is_background"):
        d = np.abs(out[k][0].cpu().numpy() - fx[k]).max()
        assert d <= TOL, "%s max abs diff %.3e" % (k, d)
    net.check_errors()


@pytest.mark.parametrize("precision,bwd_fp32", [("bf16x3", 0), ("bf16x3", 1), ("bf16x3", 4), ("fp32", 0)])
def test_gradients_match_reference_fixture(golden_dir, precision, bwd_fp32):
    fx = golden.load(golden_dir, "tiny_rw2c")
    cfg, net = _fixture_net(fx, pnb_precision=precision, pnb_bwd_fp32=bwd_fp32)
    out = _forward(net, scene.make_rays(cfg, fx["pixels"]))
    assert np.abs(out["coarse_raycolor"][0].detach().cpu().numpy() - fx["coarse_raycolor"]).max() <= TOL
    loss = (out["coarse_raycolor"] ** 2).sum() + 1e-3 * out["conf_coefficient"].sum()   # the loss of oracle/make_golden_rw2c.py
    loss.backward()
    npn = net.neural_points
    per_point = _close_points if bwd_fp32 == 0 else _close
    per_point(npn.points_embeding.grad.cpu(), fx["grad_embedding"], "points_embeding")
    per_point(npn.points_color.grad.cpu(), fx["grad_color"], "points_color")
    per_point(npn.points_dir.grad.cpu(), fx["grad_dir"], "points_dir")
    _close(npn.points_conf.grad.cpu(), fx["grad_conf"], "points_conf", rtol=1e-3)
    for k, p in net.aggregator.named_parameters():
        _close(p.grad.cpu(), fx["gradmlp." + k], "aggregator." + k, rtol=1e-3 if bwd_fp32 == 0 else 3e-4)
    assert npn.Rw2c.grad is None and npn.xyz.grad is None
    net.check_errors()


def _train_step(net, rays):
    for p in net.parameters():
        p.grad = None
    out = _forward(net, rays)
    ((out["coarse_raycolor"] ** 2).sum() + 1e-3 * out["conf_coefficient"].sum()).backward()
    grads = {k: p.grad.detach().clone() for k, p in net.named_parameters() if p.grad is not None}
    return out["coarse_raycolor"].detach().clone(), grads


# weight gradients the tensor-core backward reduces with its deterministic split-K (csrc/backward.cu, gemm_tn_acc); the biases (colsum),
# the alpha branch, colour_branch.6 and the point gradients are accumulated with atomics
DETERMINISTIC_GRADS = tuple("aggregator.%s.weight" % k for k in
                            ("block1.0", "block1.2", "block3.0", "block3.2", "color_branch.0", "color_branch.2", "color_branch.4"))


@pytest.mark.parametrize("precision", PRECISIONS)
def test_equal_rows_are_bitwise_the_uniform_path(precision):
    """Rows all equal to M: the per-point kernels read the same nine numbers per pair and evaluate the same expressions, so the
    outputs are bitwise those of Rw2c = M.  Gradients (the default tensor-core backward): bitwise where it reduces
    deterministically, within the fixture tolerance where it accumulates with atomics."""
    cfg = scene.CONFIGS["tiny"]
    M = scene.edit_frames(torch.tensor([[1.0, 0.0, 0.0]]))[0]
    net, pts, opt = harness.build_model(cfg, DEV, alpha_bias=4.0, pnb_bwd_fp32=0, **_prec(precision))
    N = pts["xyz"].shape[0]
    rays = scene.make_rays(cfg, scene.centre_patch(cfg, 48))
    _set_frames(net, M)
    uni = _render_full(net, cfg, rays)
    uni = {k: v.clone() for k, v in uni.items()}
    col_u, g_u = _train_step(net, rays)
    _set_frames(net, M.expand(N, 3, 3).contiguous())
    per = _render_full(net, cfg, rays)
    for k in uni:
        assert torch.equal(uni[k], per[k]), k
    col_p, g_p = _train_step(net, rays)
    assert torch.equal(col_u, col_p)
    assert set(g_u) == set(g_p) and "neural_points.Rw2c" not in g_p
    assert set(DETERMINISTIC_GRADS) <= set(g_u)
    for k in g_u:
        if k in DETERMINISTIC_GRADS:
            assert torch.equal(g_u[k], g_p[k]), k
        else:
            _close(g_p[k].cpu(), g_u[k].cpu(), k, rtol=1e-4)
    net.check_errors()


@pytest.mark.parametrize("precision", PRECISIONS)
def test_render_order1_matches_oracle(precision):
    """agg_intrp_order 1 (alpha_branch on the K-aggregated feature) with two objects in their own frames."""
    cfg = scene.CONFIGS["tiny"]
    net, pts, opt = harness.build_model(cfg, DEV, alpha_bias=4.0, agg_intrp_order=1, **_prec(precision))
    R = scene.edit_frames(pts["xyz"])
    _set_frames(net, R)
    rays = scene.make_rays(cfg, scene.centre_patch(cfg, 64))
    out = _render_full(net, cfg, rays)
    ref = _oracle_render(cfg, opt, pts, net.aggregator, rays["raydir"][0], R)
    assert np.array_equal(out["ray_mask"][0].cpu().numpy(), ref["ray_mask"])
    for a in ("coarse_raycolor", "coarse_point_opacity", "coarse_is_background"):
        d = (out[a][0].cpu() - ref[a]).abs().max().item()
        assert d <= TOL, "%s max abs diff %.3e" % (a, d)
    net.check_errors()


@pytest.mark.parametrize("precision", PRECISIONS)
def test_render_lego_scale(precision):
    """BASELINE config 2 size (N = 400k) with the two-object frames: a reference-sized chunk against the oracle, and the frames make
    a difference of more than the tolerance."""
    cfg = scene.CONFIGS["lego_render"]
    net, pts, opt = harness.build_model(cfg, DEV, alpha_bias=3.0, **_prec(precision))
    chunk = scene.make_rays(cfg, scene.centre_patch(cfg, 40))
    plain = _render_full(net, cfg, chunk)["coarse_raycolor"].clone()
    R = scene.edit_frames(pts["xyz"])
    _set_frames(net, R)
    out = _render_full(net, cfg, chunk)
    ref = _oracle_render(cfg, opt, pts, net.aggregator, chunk["raydir"][0], R)
    assert np.array_equal(out["ray_mask"][0].cpu().numpy(), ref["ray_mask"])
    for a in ("coarse_raycolor", "coarse_point_opacity", "coarse_is_background"):
        d = (out[a][0].cpu() - ref[a]).abs().max().item()
        assert d <= TOL, "%s max abs diff %.3e" % (a, d)
    change = (plain - out["coarse_raycolor"]).abs().max().item()
    assert change > 10 * TOL, "the frames change the chunk's radiance by only %.3e" % change
    net.check_errors()


def test_install_into_reference_shaped_module_with_per_point_frames():
    """Seam B (INTEGRATION.md) with an edited scene: the reference-shaped module keeps neural_points.Rw2c [N,3,3] as its own
    parameter (requires_grad False, neural_points.py:466-467) and the patched forward reads it in place."""
    import torch.nn as nn
    from pointnerf_b200 import ray_marching as P
    from pointnerf_b200.point_query import lighting_fast_querier

    cfg = scene.CONFIGS["tiny"]
    opt = harness.make_opt(cfg)
    pts = scene.make_points(cfg)
    R = scene.edit_frames(pts["xyz"])

    class RefNeuralPoints(nn.Module):
        def __init__(self):
            super().__init__()
            self.xyz = nn.Parameter(pts["xyz"].to(DEV), requires_grad=False)
            self.points_embeding = nn.Parameter(pts["embedding"].to(DEV))
            self.points_conf = nn.Parameter(pts["conf"].to(DEV))
            self.points_dir = nn.Parameter(pts["dir"].to(DEV))
            self.points_color = nn.Parameter(pts["color"].to(DEV))
            self.Rw2c = nn.Parameter(R.to(DEV), requires_grad=False)
            self.querier = lighting_fast_querier(torch.device(DEV), opt)

    class RefRayMarching(nn.Module):
        def __init__(self, aggregator, neural_points, opt):
            super().__init__()
            self.aggregator, self.neural_points, self.opt = aggregator, neural_points, opt

        def forward(self, *a, **k):
            raise AssertionError("the eager reference forward must have been replaced")

    P.install_into(RefRayMarching)
    agg = P.PointAggregator(opt, seed=0).to(DEV)
    with torch.no_grad():
        agg.alpha_branch[0].bias += 4.0
    net = RefRayMarching(agg, RefNeuralPoints(), opt)
    rays = scene.make_rays(cfg, scene.centre_patch(cfg, 32))
    with torch.no_grad():
        out = _forward(net, rays)
    ref = _oracle_render(cfg, opt, pts, agg, rays["raydir"][0], R)
    assert np.array_equal(out["ray_mask"][0].cpu().numpy(), ref["ray_mask"])
    assert (out["coarse_raycolor"][0].cpu() - ref["ray_color"]).abs().max().item() <= TOL


def test_bad_per_point_frames_are_refused():
    cfg = scene.CONFIGS["tiny"]
    net, pts, opt = harness.build_model(cfg, DEV, alpha_bias=4.0)
    rays = scene.make_rays(cfg, scene.centre_patch(cfg, 8))
    R = scene.edit_frames(pts["xyz"]).to(DEV)
    for bad in (R[:-1], R.double(), R.cpu(), R.transpose(1, 2), R[None]):
        net.neural_points.Rw2c = bad
        with pytest.raises(PnbError, match="Rw2c"):
            _render_full(net, cfg, rays)
