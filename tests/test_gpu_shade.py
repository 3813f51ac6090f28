"""GPU parity, floating-point path: fused shading + compositing through the C ABI against the CPU oracle
(oracle/shade_oracle.py, itself pinned to the reference's Python) and the reference-generated fixtures.
Tolerance: 1e-4 absolute on rendered radiance / opacity (BASELINE.json north_star)."""
import os

import numpy as np
import pytest
import torch

from oracle import pipeline
from pointnerf_b200 import harness, scene
from oracle import golden  # noqa: E402

pytestmark = pytest.mark.gpu
DEV = "cuda:0"
TOL = 1e-4


def _prec(precision):
    """bf16x3: the default (render_full / eval forward run the frozen-cloud pair kernel k_shade_wg<FROZEN>);
    bf16x3-general: the general pair kernel k_shade_wg (what training steps run); fp32: the exact CUDA-core kernel."""
    if precision == "bf16x3-general":
        return dict(pnb_precision="bf16x3", pnb_frozen=0)
    return dict(pnb_precision=precision)


PRECISIONS = ["bf16x3", "bf16x3-general", "fp32"]


def _oracle_render(cfg, opt, pts, agg, raydir):
    return pipeline.render(pts, harness.mlp_cpu(agg), raydir, cfg.campos, np.eye(3, dtype=np.float32), cfg.near, cfg.far,
                           opt.vsize, opt.vscale, opt.kernel_size, opt.query_size, opt.ranges, opt.SR, opt.K, opt.P,
                           opt.max_o if opt.max_o is not None else pts["xyz"].shape[0], D=cfg.D)


def _render_full(net, cfg, rays):
    with torch.no_grad():
        return net.render_full(list(cfg.campos), rays["raydir"].to(DEV), torch.eye(3), cfg.near, cfg.far, [1., 1., 1.])


@pytest.mark.parametrize("precision", PRECISIONS)
@pytest.mark.parametrize("name,side,alpha_bias,over", [
    ("tiny", 64, 4.0, {}), ("tiny", 64, 0.0, {}), ("tiny", 40, 8.0, dict(SR=8)), ("tiny", 40, 4.0, dict(K=3)),
    ("chair_plumbing", 16, 4.0, {}), ("chair_plumbing", 64, 2.0, dict(SR=80)),
])
def test_render_matches_oracle(name, side, alpha_bias, over, precision):
    cfg = scene.CONFIGS[name]
    net, pts, opt = harness.build_model(cfg, DEV, alpha_bias=alpha_bias, **_prec(precision), **over)
    rays = scene.make_rays(cfg, scene.centre_patch(cfg, side))
    out = _render_full(net, cfg, rays)
    ref = _oracle_render(cfg, opt, pts, net.aggregator, rays["raydir"][0])
    assert np.array_equal(out["ray_mask"][0].cpu().numpy(), ref["ray_mask"])
    for a in ("coarse_raycolor", "coarse_point_opacity", "coarse_is_background"):
        d = (out[a][0].cpu() - ref[a]).abs().max().item()
        assert d <= TOL, "%s max abs diff %.3e" % (a, d)
    assert ref["coarse_is_background"].min() < 0.9 or alpha_bias == 0.0   # the case is not trivially transparent
    net.check_errors()


@pytest.mark.parametrize("precision", PRECISIONS)
@pytest.mark.parametrize("name", ["tiny_opaque", "tiny_thin_sr8", "tiny_order1", "tiny_raydist0_bg"])
def test_forward_matches_reference_fixture(name, golden_dir, precision):
    """The drop-in NeuralPointsRayMarching.forward() output dict vs what the reference module itself returned
    (tiny_order1: the reference run with --agg_intrp_order 1, SURVEY 8(f) rank 4; tiny_raydist0_bg: with --raydist_mode_unit 0 and
    bg_color (0.9, 0.1, 0.4))."""
    fx = golden.load(golden_dir, name)
    cfg = scene.CONFIGS["tiny"]
    order = int(fx["agg_intrp_order"]) if "agg_intrp_order" in fx.files else 2
    mode_unit = int(fx["raydist_mode_unit"]) if "raydist_mode_unit" in fx.files else 1
    net, pts, opt = harness.build_model(cfg, DEV, SR=int(fx["SR"]), max_o=100000, agg_intrp_order=order, raydist_mode_unit=mode_unit,
                                        **_prec(precision))
    sd = {k[4:]: torch.from_numpy(fx[k]) for k in fx.files if k.startswith("mlp.")}
    net.aggregator.load_state_dict(sd)
    rays = scene.make_rays(cfg, fx["pixels"], bg_color=fx["bg_color"].tolist() if "bg_color" in fx.files else (1.0, 1.0, 1.0))
    r = {k: v.to(DEV) for k, v in rays.items()}
    with torch.no_grad():
        out = net(r["campos"], r["raydir"], bg_color=r["bg_color"], camrotc2w=r["camrotc2w"], pixel_idx=r["pixel_idx"],
                  near=r["near"], far=r["far"], h=r["h"], w=r["w"], intrinsic=r["intrinsic"])
    assert np.array_equal(out["ray_mask"][0].cpu().numpy(), fx["ray_mask"])
    for k in ("coarse_raycolor", "coarse_point_opacity", "coarse_is_background"):
        d = np.abs(out[k][0].cpu().numpy() - fx[k]).max()
        assert d <= TOL, "%s max abs diff %.3e" % (k, d)
    assert out["queried_shading"].shape == (1, fx["sample_pidx"].shape[0], 3)
    # exactly the keys (and trailing shapes) the reference module returns in evaluation mode (tests/golden/output_keys.json,
    # generated from the reference's own forward by oracle/make_golden.py)
    import json
    want = json.load(open(os.path.join(golden_dir, "output_keys.json")))["eval"]
    assert sorted(out.keys()) == sorted(want.keys())
    for k, tail in want.items():
        exp = [int(fx["SR"]) if (d == 24 and k != "coarse_raycolor") else d for d in tail]
        assert list(out[k].shape[2:]) == exp, (k, list(out[k].shape), exp)


@pytest.mark.parametrize("precision", PRECISIONS)
@pytest.mark.parametrize("name,side,over", [("tiny", 64, {}), ("chair_plumbing", 48, dict(SR=80)), ("lego_render", 40, {})])
def test_render_order1_matches_oracle(name, side, over, precision):
    """agg_intrp_order = 1 (point_aggregators.py:573-599: alpha_branch on the K-aggregated feature) through render_full, all three
    kernels (frozen / general wgmma pair kernels, fp32), against the oracle (itself pinned to the reference run of tiny_order1.npz)."""
    cfg = scene.CONFIGS[name]
    net, pts, opt = harness.build_model(cfg, DEV, alpha_bias=3.0, agg_intrp_order=1, **_prec(precision), **over)
    rays = scene.make_rays(cfg, scene.centre_patch(cfg, side))
    out = _render_full(net, cfg, rays)
    ref = pipeline.render(pts, harness.mlp_cpu(net.aggregator), rays["raydir"][0], cfg.campos, np.eye(3, dtype=np.float32), cfg.near, cfg.far,
                          opt.vsize, opt.vscale, opt.kernel_size, opt.query_size, opt.ranges, opt.SR, opt.K, opt.P, pts["xyz"].shape[0], D=cfg.D,
                          agg_intrp_order=1)
    assert np.array_equal(out["ray_mask"][0].cpu().numpy(), ref["ray_mask"])
    for a in ("coarse_raycolor", "coarse_point_opacity", "coarse_is_background"):
        d = (out[a][0].cpu() - ref[a]).abs().max().item()
        assert d <= TOL, "%s max abs diff %.3e" % (a, d)
    ref2 = _oracle_render(cfg, opt, pts, net.aggregator, rays["raydir"][0])          # and order 1 is not order 2 on this case
    assert (ref2["coarse_point_opacity"] - ref["coarse_point_opacity"]).abs().max().item() > 10 * TOL
    net.check_errors()


@pytest.mark.parametrize("precision", PRECISIONS)
def test_render_lego_scale(precision):
    """BASELINE config 2 size: a reference-sized chunk against the oracle; full-frame determinism and
    sharding invariance (bit-exact: a ray's colour does not depend on which rays share the call)."""
    cfg = scene.CONFIGS["lego_render"]
    net, pts, opt = harness.build_model(cfg, DEV, alpha_bias=3.0, **_prec(precision))
    chunk = scene.make_rays(cfg, scene.centre_patch(cfg, 40))
    out = _render_full(net, cfg, chunk)
    ref = _oracle_render(cfg, opt, pts, net.aggregator, chunk["raydir"][0])
    assert np.array_equal(out["ray_mask"][0].cpu().numpy(), ref["ray_mask"])
    for a in ("coarse_raycolor", "coarse_point_opacity", "coarse_is_background"):
        d = (out[a][0].cpu() - ref[a]).abs().max().item()
        assert d <= TOL, "%s max abs diff %.3e" % (a, d)
    full = scene.make_rays(cfg)
    a = _render_full(net, cfg, full)
    col_a, op_a = a["coarse_raycolor"].clone(), a["coarse_point_opacity"].clone()
    b = _render_full(net, cfg, full)
    assert torch.equal(col_a, b["coarse_raycolor"]) and torch.equal(op_a, b["coarse_point_opacity"])
    R = full["raydir"].shape[1]
    for g in range(2):
        sel = torch.arange(g, R, 2)
        part = dict(full); part["raydir"] = full["raydir"][:, sel]
        c = _render_full(net, cfg, part)
        assert torch.equal(c["coarse_raycolor"][0], col_a[0][sel.to(DEV)])
    hit = (a["ray_mask"][0] > 0)
    assert torch.all(col_a[0][~hit] == 1.0) and torch.all(op_a[0][~hit] == 0)
    assert torch.isfinite(col_a).all() and col_a.min() >= -0.002 and col_a.max() <= 1.002
    net.check_errors()


@pytest.mark.parametrize("name,side", [("truck_8gpu", 24), ("scannet_8gpu", 16)])
def test_render_large_configs_chunk(name, side):
    """BASELINE configs 4/5 sizes: rendered radiance of a chunk vs the oracle (default wgmma path)."""
    cfg = scene.CONFIGS[name]
    net, pts, opt = harness.build_model(cfg, DEV, alpha_bias=3.0)
    rays = scene.make_rays(cfg, scene.centre_patch(cfg, side))
    out = _render_full(net, cfg, rays)
    ref = _oracle_render(cfg, opt, pts, net.aggregator, rays["raydir"][0])
    assert np.array_equal(out["ray_mask"][0].cpu().numpy(), ref["ray_mask"])
    for a in ("coarse_raycolor", "coarse_point_opacity", "coarse_is_background"):
        d = (out[a][0].cpu() - ref[a]).abs().max().item()
        assert d <= TOL, "%s max abs diff %.3e" % (a, d)
    net.check_errors()


def _block(x0, y0, w, h):
    px, py = np.meshgrid(np.arange(x0, x0 + w), np.arange(y0, y0 + h))
    return np.stack((px, py), -1).reshape(-1, 2).astype(np.float32)


@pytest.mark.parametrize("precision", ["bf16x3", "bf16x3-general"])
@pytest.mark.parametrize("name,block,over", [
    ("lego_render", (640, 388, 96, 24), {}),                 # through the limb of the shell: grazing hits, partial neighbourhoods, misses
    ("lego_render", (640, 388, 96, 24), dict(SR=80)),        # the shipped SR
    ("truck_8gpu", (860, 0, 100, 16), {}),                   # image corner: the limb crosses the strip (kernel_size 5)
    ("scannet_8gpu", (0, 228, 64, 24), {}),                  # left image edge across a wall/wall corner of the box, all rays hit
])
def test_render_silhouette_strips(name, block, over, precision):
    """Oracle parity where neighbourhoods are partial (silhouette-crossing strips at the BASELINE sizes)."""
    cfg = scene.CONFIGS[name]
    net, pts, opt = harness.build_model(cfg, DEV, alpha_bias=3.0, **_prec(precision), **over)
    rays = scene.make_rays(cfg, _block(*block))
    out = _render_full(net, cfg, rays)
    ref = _oracle_render(cfg, opt, pts, net.aggregator, rays["raydir"][0])
    m = ref["ray_mask"]
    assert np.array_equal(out["ray_mask"][0].cpu().numpy(), m)
    if name != "scannet_8gpu":
        assert 0 < int(m.sum()) < m.size, "the strip must cross the silhouette"
    for a in ("coarse_raycolor", "coarse_point_opacity", "coarse_is_background"):
        d = (out[a][0].cpu() - ref[a]).abs().max().item()
        assert d <= TOL, "%s max abs diff %.3e" % (a, d)
    net.check_errors()


def _pack_reference(counts, PACK_S=512, PACK_WIN=64):
    """Python restatement of k_pack_quads (same as tests/test_host_logic.py): first fit with a look-ahead window, per super-chunk."""
    vorder, vcntp, qf = [], [], []
    for i0 in range(0, len(counts), PACK_S):
        c = list(counts[i0:i0 + PACK_S])
        n, pos, emitted = len(c), 0, 0
        while pos < n:
            qf.append(i0 + emitted)
            rows = 0
            for i in range(pos, min(n, pos + PACK_WIN)):
                if rows >= 32:
                    break
                if c[i] != 0 and rows + c[i] <= 32:
                    vorder.append(i0 + i); vcntp.append(c[i]); rows += c[i]; c[i] = 0; emitted += 1
            while pos < n and c[pos] == 0:
                pos += 1
    qf.append(len(counts))
    return np.array(vorder), np.array(vcntp), np.array(qf)


@pytest.mark.parametrize("name,side", [("tiny", 64), ("chair_plumbing", 200), ("lego_render", 300)])
def test_row_packing_tables_match_restatement(name, side):
    """The warp-cooperative packing kernels produce exactly the tables of the sequential first-fit algorithm."""
    import ctypes as C
    from pointnerf_b200 import lib as L
    cfg = scene.CONFIGS[name]
    net, pts, opt = harness.build_model(cfg, DEV, alpha_bias=3.0)
    rays = scene.make_rays(cfg, scene.centre_patch(cfg, side))
    _render_full(net, cfg, rays)
    net.check_errors()
    q = net.last
    cnt = q.counters_tensor().cpu().numpy()
    n_valid = int(cnt[L.QC["n_valid"]])
    assert n_valid > 1000
    ws = q.ws
    def view(ptr, nbytes, dtype):
        off = int(ptr) - ws.data_ptr()
        return ws[off:off + nbytes].view(dtype)
    valid_list = view(q.desc.valid_list, 4 * n_valid, torch.int32).cpu().numpy()
    nv = view(q.desc.samp_nvalid, int(cnt[L.QC["n_cand"]]), torch.uint8).cpu().numpy()
    counts = nv[valid_list].astype(np.int64)
    ptrs = [C.c_void_p() for _ in range(4)]
    L.check(L.load().pnb_shade_tc_tables(net._tc_ws.data_ptr(), net._tc_ws.numel(), net._max_valid, *[C.byref(p) for p in ptrs]), "tables")
    def tview(ptr, nbytes, dtype):
        off = ptr.value - net._tc_ws.data_ptr()
        return net._tc_ws[off:off + nbytes].view(dtype).cpu().numpy()
    n_quads = int(tview(ptrs[3], 4, torch.int32)[0])
    vorder = tview(ptrs[0], 4 * n_valid, torch.int32)
    vcntp = tview(ptrs[1], n_valid, torch.uint8)
    qf = tview(ptrs[2], 4 * (n_quads + 1), torch.int32)
    rv, rc, rq = _pack_reference(counts)
    assert n_quads == len(rq) - 1
    assert np.array_equal(vorder, rv) and np.array_equal(vcntp, rc) and np.array_equal(qf, rq)
    rows = np.add.reduceat(rc, rq[:-1])
    assert rows.max() <= 32 and rows.sum() == counts.sum()


def test_frozen_table_follows_parameter_updates():
    """The hoisted per-point table of the frozen pipeline is rebuilt when points_embeding or block1.0 change in place."""
    cfg = scene.CONFIGS["tiny"]
    net, pts, opt = harness.build_model(cfg, DEV, alpha_bias=4.0)
    gen, _, _ = harness.build_model(cfg, DEV, alpha_bias=4.0, pnb_frozen=0)
    rays = scene.make_rays(cfg, scene.centre_patch(cfg, 48))
    a0 = _render_full(net, cfg, rays)["coarse_raycolor"].clone()
    g0 = _render_full(gen, cfg, rays)["coarse_raycolor"].clone()
    assert (a0 - g0).abs().max().item() <= 2e-5
    with torch.no_grad():
        for m in (net, gen):
            m.neural_points.points_embeding.mul_(0.5)
            m.aggregator.block1[0].weight.mul_(1.1)
            m.aggregator.block1[0].bias.add_(0.01)
    a1 = _render_full(net, cfg, rays)["coarse_raycolor"]
    g1 = _render_full(gen, cfg, rays)["coarse_raycolor"]
    assert (a1 - a0).abs().max().item() > 1e-3                      # the update is visible ...
    assert (a1 - g1).abs().max().item() <= 2e-5                     # ... and the frozen path tracks the general one


@pytest.mark.parametrize("name,side,over", [("tiny", 64, {}), ("lego_render", 96, {}), ("lego_render", 64, dict(SR=80)), ("truck_8gpu", 48, {})])
def test_persistent_tile_loop_is_bit_identical(name, side, over):
    """The pair and colour kernels on one CTA per 8 SMs (pnb_dbg_flags bit 3: many tiles per persistent CTA, the weight ring running
    across tile boundaries) against the default launch (one CTA per SM): the same arithmetic per tile -> equal bits."""
    cfg = scene.CONFIGS[name]
    a, _, _ = harness.build_model(cfg, DEV, alpha_bias=3.0, **over)
    b, _, _ = harness.build_model(cfg, DEV, alpha_bias=3.0, pnb_dbg_flags=8, **over)
    rays = scene.make_rays(cfg, scene.centre_patch(cfg, side))
    for rep in range(2):
        oa, ob = _render_full(a, cfg, rays), _render_full(b, cfg, rays)
        a.check_errors(); b.check_errors()
        for k in ("coarse_raycolor", "coarse_point_opacity", "coarse_is_background"):
            assert torch.equal(oa[k], ob[k]), k
    assert oa["coarse_point_opacity"].max().item() > 0.0             # the patch is not empty space


def test_workspace_overflow_is_safe_and_reported():
    """A frame denser than the workspace heuristic (indoor scene: every ray keeps all SR samples): the dropped samples contribute
    nothing (no uninitialised reads), the call is reported (check_errors / the next call), and the retry is exact."""
    from pointnerf_b200 import lib as L, runner
    cfg = scene.CONFIGS["scannet_8gpu"]
    net, pts, opt = harness.build_model(cfg, DEV, alpha_bias=3.0, pnb_max_valid_per_ray=2)
    rays = scene.make_rays(cfg)                                          # 307,200 rays, every one hits a wall: several valid samples per ray >> 2
    out = _render_full(net, cfg, rays)
    col = out["coarse_raycolor"].clone()
    assert torch.isfinite(col).all() and col.min() >= -0.002 and col.max() <= 1.002
    n_valid = int(net.last.counters_tensor()[L.QC["n_valid"]].item())
    assert n_valid > net._max_valid, "the test frame must overflow the workspace (%d valid samples, capacity %d)" % (n_valid, net._max_valid)
    with pytest.raises(L.PnbOverflow):
        net.check_errors()
    out2 = _render_full(net, cfg, rays)                                  # the workspace grew: exact now
    net.check_errors()
    col2 = out2["coarse_raycolor"]
    chunk = dict(rays); chunk["raydir"] = rays["raydir"][:, :4096]
    ref = _render_full(net, cfg, chunk)["coarse_raycolor"]
    assert torch.equal(col2[:, :4096], ref)
    assert not torch.equal(col, col2)
    # the whole-image entry checks and retries by itself
    net3, _, _ = harness.build_model(cfg, DEV, alpha_bias=3.0, pnb_max_valid_per_ray=2)
    data = {k: (v.to(DEV) if isinstance(v, torch.Tensor) else v) for k, v in rays.items()}
    img = runner.render_image(net3, data, cfg.H, cfg.W)
    assert torch.equal(img["coarse_raycolor"].reshape(1, -1, 3), col2)
    # deferred report: without check_errors() the NEXT call raises
    net4, _, _ = harness.build_model(cfg, DEV, alpha_bias=3.0, pnb_max_valid_per_ray=2)
    _render_full(net4, cfg, rays)
    torch.cuda.synchronize()
    with pytest.raises(L.PnbOverflow):
        _render_full(net4, cfg, rays)


def test_probe_outputs_match_reference_fixture(golden_dir):
    """opt.prob == 1 (point-growing probe, run/train_ft.py:417-530): the extra per-ray outputs of the drop-in forward
    vs what the reference module returned (neural_points_volumetric_model.py:331-351)."""
    fx = np.load(os.path.join(golden_dir, "tiny_probe.npz"))
    wfx = golden.load(golden_dir, "tiny_opaque")
    cfg = scene.CONFIGS["tiny"]
    net, pts, opt = harness.build_model(cfg, DEV, max_o=100000, prob=1)
    net.aggregator.load_state_dict({k[4:]: torch.from_numpy(wfx[k]) for k in wfx.files if k.startswith("mlp.")})
    rays = scene.make_rays(cfg, fx["pixels"])
    r = {k: v.to(DEV) for k, v in rays.items()}
    with torch.no_grad():
        out = net(r["campos"], r["raydir"], bg_color=r["bg_color"], camrotc2w=r["camrotc2w"], pixel_idx=r["pixel_idx"],
                  near=r["near"], far=r["far"], h=r["h"], w=r["w"], intrinsic=r["intrinsic"])
    # rays whose arg-max opacity is (numerically) tied between two samples may pick the other sample: compare where
    # the selected sample location agrees, and require that to be (almost) everywhere
    import json
    assert sorted(out.keys()) == sorted(json.load(open(os.path.join(golden_dir, "output_keys.json")))["probe"].keys())
    loc = out["ray_max_sample_loc_w"][0].cpu().numpy()
    same = np.abs(loc - fx["ray_max_sample_loc_w"]).max(-1) == 0
    assert same.mean() > 0.98
    for k, tol in (("ray_max_shading_opacity", 1e-4), ("ray_max_far_dist", 1e-6), ("shading_avg_color", 1e-5),
                   ("shading_avg_dir", 1e-5), ("shading_avg_conf", 1e-5), ("shading_avg_embedding", 1e-5)):
        a = out[k][0].cpu().numpy().reshape(fx[k].shape)
        assert np.abs(a - fx[k])[same].max() <= tol, k


def test_install_into_reference_shaped_module():
    """Seam B (INTEGRATION.md): patching a reference-shaped NeuralPointsRayMarching class (own parameters under
    self.neural_points / self.aggregator, reference attribute names) with install_into() gives the fused forward."""
    import torch.nn as nn
    from pointnerf_b200 import ray_marching as P
    from pointnerf_b200.point_query import lighting_fast_querier

    cfg = scene.CONFIGS["tiny"]
    opt = harness.make_opt(cfg)
    pts = scene.make_points(cfg)

    class RefNeuralPoints(nn.Module):            # attribute names of models/neural_points/neural_points.py
        def __init__(self):
            super().__init__()
            self.xyz = nn.Parameter(pts["xyz"].to(DEV), requires_grad=False)
            self.points_embeding = nn.Parameter(pts["embedding"].to(DEV))
            self.points_conf = nn.Parameter(pts["conf"].to(DEV))
            self.points_dir = nn.Parameter(pts["dir"].to(DEV))
            self.points_color = nn.Parameter(pts["color"].to(DEV))
            self.Rw2c = torch.eye(3, device=DEV)
            self.querier = lighting_fast_querier(torch.device(DEV), opt)      # seam A

    class RefRayMarching(nn.Module):             # stands in for models.neural_points_volumetric_model.NeuralPointsRayMarching
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
    r = {k: v.to(DEV) for k, v in rays.items()}
    with torch.no_grad():
        out = net(r["campos"], r["raydir"], bg_color=r["bg_color"], camrotc2w=r["camrotc2w"], pixel_idx=r["pixel_idx"],
                  near=r["near"], far=r["far"], h=r["h"], w=r["w"], intrinsic=r["intrinsic"])
    ref = _oracle_render(cfg, opt, pts, agg, rays["raydir"][0])
    assert np.array_equal(out["ray_mask"][0].cpu().numpy(), ref["ray_mask"])
    assert (out["coarse_raycolor"][0].cpu() - ref["ray_color"]).abs().max().item() <= TOL
    assert sorted(k for k, _ in net.named_parameters())[:3] == ["aggregator.alpha_branch.0.bias", "aggregator.alpha_branch.0.weight",
                                                                 "aggregator.block1.0.bias"]
