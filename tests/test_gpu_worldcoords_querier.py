"""GPU: the world-coordinate querier of wcoord_query 1 (pointnerf_b200.query_point_indices_worldcoords), which reads its query options
from opt on every call, against the wcoord_query -1 querier (options read once, at construction) and oracle/query_oracle.

  options unchanged   over a 2304-ray chunk loop (the reference's chunk size) the 7-tuple of query_points is bit for bit the -1
                      querier's, and the grid is built once (tiny, lego centre, truck with kernel 5)
  options changed     after each change (query_size 3 -> 1, kernel_size, vsize, radius_limit_scale, ranges) the 7-tuple is bit for bit a
                      freshly constructed -1 querier's with the new options and the oracle's (ray mask, slots, counters); an option the
                      grid depends on rebuilds it exactly once, radius_limit_scale (the query's alone) and an unchanged call never do
  fused module        with wcoord_query 1, after `opt.query_size = [1, 1, 1]` (what probe_hole does between its probe tiers) probe_image,
                      render_image and forward() are bit for bit a module built with query size 1 1 1; probe_image equals the 2304-ray
                      chunk loop; one training step's gradients agree with that module's within oracle/grad_check.RTOL (the backward's
                      atomic sums differ in order between runs); with options unchanged every output is the wcoord_query -1 module's
"""
import copy

import numpy as np
import pytest
import torch

from oracle import grad_check, pipeline, query_oracle
from pointnerf_b200 import harness, runner, scene
from pointnerf_b200 import point_query as wq
from pointnerf_b200 import query_point_indices_worldcoords as wc

pytestmark = pytest.mark.gpu
DEV = "cuda:0"
CHUNK = 2304


def _rays(cfg, pixels=None, rotated=False):
    r = scene.make_rays(cfg, pixels, camrotc2w=scene.orbit_rotation() if rotated else None)
    return {k: (v.to(DEV) if isinstance(v, torch.Tensor) else v) for k, v in r.items()}


def _query(q, xyz, r, start=0, end=None):
    return q.query_points(r["pixel_idx"][:, start:end].to(torch.int32), None, xyz[None], None, 0, 0, None, np.float32(r["near"].item()),
                          np.float32(r["far"].item()), r["raydir"][:, start:end].contiguous(), r["campos"], r["camrotc2w"])


def _assert_same_tuple(a, b, tag=""):
    assert len(a) == len(b) == 7
    for i in range(5):
        assert a[i].dtype == b[i].dtype and a[i].shape == b[i].shape and torch.equal(a[i], b[i]), (tag, i)
    assert list(a[5]) == list(b[5]) and np.array_equal(a[6], b[6]), tag


@pytest.mark.parametrize("name,side", [("tiny", None), ("lego_render", 96), ("truck_8gpu", 96)])
def test_unchanged_options_are_the_minus_one_querier_over_a_chunk_loop(name, side):
    cfg = scene.CONFIGS[name]
    opt = harness.make_opt(cfg, wcoord_query=1)
    xyz = scene.make_points(cfg)["xyz"].to(DEV).contiguous()
    r = _rays(cfg, None if side is None else scene.centre_patch(cfg, side))
    ours, ref = wc.lighting_fast_querier(torch.device(DEV), opt), wq.lighting_fast_querier(torch.device(DEV), opt)
    R = r["raydir"].shape[1]
    assert R > CHUNK
    hits = 0
    for start in range(0, R, CHUNK):
        a, b = _query(ours, xyz, r, start, start + CHUNK), _query(ref, xyz, r, start, start + CHUNK)
        _assert_same_tuple(a, b, (name, start))
        assert a[5] is opt.vsize
        hits += int(a[4].sum())
    assert hits > 0
    assert ours.n_builds == 1 and ref.n_builds == 1


def _oracle(cfg, opt, xyz_cpu, raydir):
    rng6, svs, dim = pipeline.hyperparameters(xyz_cpu, opt.vsize, opt.vscale, opt.kernel_size, opt.ranges)
    return query_oracle.query(xyz_cpu.numpy(), rng6[:3], svs, dim, opt.kernel_size, opt.query_size,
                              opt.max_o if opt.max_o is not None else xyz_cpu.shape[0], opt.P,
                              float(pipeline.radius_limit(opt.radius_limit_scale, opt.vsize)),
                              campos=np.array(cfg.campos, np.float32), raydir=raydir.cpu().numpy(), t=pipeline.t_table(cfg.near, cfg.far, cfg.D),
                              SR=opt.SR, K=opt.K)


@pytest.mark.parametrize("name,side", [("tiny", 48), ("lego_render", 48)])
def test_changed_options_are_a_fresh_minus_one_querier_and_the_oracle(name, side):
    cfg = scene.CONFIGS[name]
    opt = harness.make_opt(cfg, wcoord_query=1)
    xyz_cpu = scene.make_points(cfg)["xyz"]
    xyz = xyz_cpu.to(DEV).contiguous()
    r = _rays(cfg, scene.centre_patch(cfg, side))
    q = wc.lighting_fast_querier(torch.device(DEV), opt)
    lo = [v for v in opt.ranges[:3]]
    hi = [v for v in opt.ranges[3:]]
    changes = [("initial", {}, 1), ("query_size 3 -> 1", dict(query_size=[1, 1, 1]), 1),
               ("kernel_size", dict(kernel_size=[5, 5, 5]), 1), ("vsize", dict(vsize=[v * 1.25 for v in opt.vsize]), 1),
               ("radius_limit_scale", dict(radius_limit_scale=2.0), 0),
               ("ranges", dict(ranges=[lo[0], lo[1], lo[2] + 0.5 * cfg.R_s, hi[0], hi[1] - 0.25 * cfg.R_s, hi[2]]), 1)]
    builds = 0
    for what, over, rebuilds in changes:
        for k, v in over.items():
            setattr(opt, k, v)
        got = _query(q, xyz, r)
        builds += rebuilds
        assert q.n_builds == builds, what
        assert _query(q, xyz, r) is not None and q.n_builds == builds, what + ": an unchanged call rebuilt the grid"
        fresh = wq.lighting_fast_querier(torch.device(DEV), copy.deepcopy(opt))
        want = _query(fresh, xyz, r)
        _assert_same_tuple(got, want, what)
        o = _oracle(cfg, opt, xyz_cpu, r["raydir"][0])
        assert np.array_equal(got[4][0].cpu().numpy(), o["ray_mask"]), what
        assert np.array_equal(got[0][0].cpu().numpy(), o["sample_pidx"]), what
        assert np.array_equal(got[2][0].cpu().numpy(), o["sample_loc_w"]), what
        gc, qc, oc = q.last_grid_counters, q.last_query_counters, o["counters"]
        for k in ("n_occ", "max_pts", "overflow_o", "overflow_p", "slot0_cell"):
            assert gc[k] == oc[k], (what, k)
        assert (qc["R1"], qc["R2"], qc["n_pairs"], qc["n_valid"]) == (oc["R1"], oc["R2"], oc["n_valid_pairs"], oc["n_valid_samples"]), what
        assert qc["R2"] > 0, what


# ------------------------------------------------------------------------------------------------------------ the fused module
def _net(cfg, **over):
    net, _, opt = harness.build_model(cfg, DEV, alpha_bias=3.0, seed=2, prob=1, **over)
    return net


def _forward(net, r, start=0, end=None):
    return net(r["campos"], r["raydir"][:, start:end], bg_color=r["bg_color"], camrotc2w=r["camrotc2w"],
               pixel_idx=r["pixel_idx"][:, start:end], near=r["near"], far=r["far"], h=r["h"], w=r["w"], intrinsic=r["intrinsic"])


def _assert_same_dict(a, b, tag):
    assert sorted(a) == sorted(b), tag
    for k in a:
        if isinstance(a[k], torch.Tensor):
            assert a[k].dtype == b[k].dtype and a[k].shape == b[k].shape and torch.equal(a[k], b[k]), (tag, k)


def _assert_same_outputs(net, ref, cfg, r):
    _assert_same_dict(runner.probe_image(net, r, cfg.H, cfg.W), runner.probe_image(ref, r, cfg.H, cfg.W), "probe_image")
    _assert_same_dict(runner.render_image(net, r, cfg.H, cfg.W), runner.render_image(ref, r, cfg.H, cfg.W), "render_image")
    with torch.no_grad():
        _assert_same_dict(_forward(net, r, 0, CHUNK), _forward(ref, r, 0, CHUNK), "forward")


def _train_step_grads(net, r):
    for p in net.parameters():
        p.grad = None
    out = _forward(net, r, 0, CHUNK)
    target = torch.full_like(out["coarse_raycolor"], 0.5)
    loss = ((out["coarse_raycolor"] - target) ** 2).mean() + 1e-3 * out["conf_coefficient"].sum() \
        + 1e-2 * out["coarse_point_opacity"].mean()
    loss.backward()
    torch.cuda.synchronize()
    net.check_errors()
    return {n: p.grad.detach().cpu().numpy() for n, p in net.named_parameters() if p.grad is not None}


def test_fused_module_follows_a_query_size_set_between_calls():
    cfg = scene.CONFIGS["tiny"]
    r = _rays(cfg, rotated=True)
    net = _net(cfg, wcoord_query=1)
    ref1 = _net(cfg, wcoord_query=-1, query_size=[1, 1, 1])
    q = net.neural_points.querier
    assert type(q) is wc.lighting_fast_querier
    runner.render_image(net, r, cfg.H, cfg.W)                           # a step at the first tier
    assert q.n_builds == 1
    net.opt.query_size = [1, 1, 1]                                      # probe_hole's tier change (run/train_ft.py:425-429)
    _assert_same_outputs(net, ref1, cfg, r)                             # probe, then the steps after it keep the tier
    assert q.n_builds == 2
    maps = runner.probe_image(net, r, cfg.H, cfg.W)
    chunked = runner.probe_image_chunked(net, r, cfg.H, cfg.W, CHUNK)
    assert sorted(maps) == sorted(chunked)
    for k in maps:
        assert maps[k].dtype == chunked[k].dtype and torch.equal(maps[k], chunked[k]), k
    assert q.n_builds == 2
    # a training step on the new tier: the same query and shading; the backward's atomic sums make the gradients close, not equal
    g, g_ref = _train_step_grads(net, r), _train_step_grads(ref1, r)
    assert sorted(g) == sorted(g_ref) and len(g) == 4 + 18
    rtol_points, rtol_mlp = grad_check.RTOL[(0, "bf16x3")]
    for n in g:
        if n.startswith("neural_points."):
            grad_check.check_points(g[n], g_ref[n], n, rtol_points)
        else:
            assert grad_check.rel_error(g[n], g_ref[n]) <= rtol_mlp, n
    # the query size differs from the first tier's: the outputs do too (the test is not vacuous)
    ref3 = _net(cfg, wcoord_query=-1)
    assert not torch.equal(runner.render_image(net, r, cfg.H, cfg.W)["coarse_raycolor"],
                           runner.render_image(ref3, r, cfg.H, cfg.W)["coarse_raycolor"])


@pytest.mark.parametrize("name,rotated", [("tiny", True), ("chair_plumbing", False)])
def test_fused_module_with_unchanged_options_is_wcoord_query_minus_one(name, rotated):
    cfg = scene.CONFIGS[name]
    r = _rays(cfg, rotated=rotated)
    net, ref = _net(cfg, wcoord_query=1), _net(cfg, wcoord_query=-1)
    _assert_same_outputs(net, ref, cfg, r)
    assert net.neural_points.querier.n_builds == 1
