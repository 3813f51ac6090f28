"""GPU parity, integer path: CUDA grid build + march + K-NN (through the C ABI, via the drop-in
lighting_fast_querier) against the CPU oracle (oracle/query_oracle.c) and the reference-generated fixtures.
Bar: ray masks, neighbour index sets and world sample positions BIT-EXACT; perspective coords 1e-6."""
import os

import numpy as np
import pytest
import torch

from oracle import pipeline, query_oracle
from pointnerf_b200 import harness, scene
from pointnerf_b200.point_query import device_t_table_jitter
from oracle import golden  # noqa: E402

pytestmark = pytest.mark.gpu
DEV = "cuda:0"


def _oracle(cfg, opt, pts, raydir, t=None):
    rng6, svs, dim = pipeline.hyperparameters(pts["xyz"], opt.vsize, opt.vscale, opt.kernel_size, opt.ranges)
    if t is None:
        t = pipeline.t_table(cfg.near, cfg.far, cfg.D)
    return query_oracle.query(pts["xyz"].numpy(), rng6[:3], svs, dim, opt.kernel_size, opt.query_size,
                              opt.max_o if opt.max_o is not None else pts["xyz"].shape[0], opt.P,
                              float(pipeline.radius_limit(opt.radius_limit_scale, opt.vsize)),
                              campos=np.array(cfg.campos, np.float32), raydir=raydir.numpy(), t=t, SR=opt.SR, K=opt.K)


def _query_points(net, rays):
    npnts = net.neural_points
    dev = torch.device(DEV)
    return npnts.querier.query_points(
        rays["pixel_idx"].to(dev).to(torch.int32), None, npnts.xyz[None], None, 0, 0, None,
        np.float32(rays["near"].item()), np.float32(rays["far"].item()), rays["raydir"].to(dev),
        rays["campos"].to(dev), rays["camrotc2w"].to(dev))


def _assert_same(out, o):
    pidx, loc, loc_w, dirs, mask = out[0][0].cpu().numpy(), out[1][0].cpu().numpy(), out[2][0].cpu().numpy(), out[3][0].cpu().numpy(), out[4][0].cpu().numpy()
    assert np.array_equal(mask, o["ray_mask"])
    assert pidx.shape == o["sample_pidx"].shape
    assert np.array_equal(np.sort(pidx, -1), np.sort(o["sample_pidx"], -1)), "neighbour index sets differ"
    assert np.array_equal(pidx, o["sample_pidx"]), "canonical K-slot order differs"
    assert np.array_equal(loc_w, o["sample_loc_w"])
    return pidx, loc, loc_w, dirs, mask


@pytest.mark.parametrize("name,side,over", [
    ("tiny", 64, {}), ("tiny", 33, dict(K=3, SR=5)), ("tiny", 40, dict(P=2)), ("tiny", 40, dict(SR=128)),
    ("chair_plumbing", 16, {}), ("chair_plumbing", 96, dict(SR=80)),
])
def test_query_matches_oracle(name, side, over):
    cfg = scene.CONFIGS[name]
    net, pts, opt = harness.build_model(cfg, DEV, **over)
    rays = scene.make_rays(cfg, scene.centre_patch(cfg, side))
    out = _query_points(net, rays)
    o = _oracle(cfg, opt, pts, rays["raydir"][0])
    pidx, loc, loc_w, dirs, mask = _assert_same(out, o)
    gc, qc, oc = net.neural_points.querier.last_grid_counters, net.neural_points.querier.last_query_counters, o["counters"]
    assert gc["n_occ"] == oc["n_occ"] and gc["max_pts"] == oc["max_pts"] and gc["overflow_p"] == oc["overflow_p"]
    assert gc["slot0_cell"] == oc["slot0_cell"]
    assert qc["R1"] == oc["R1"] and qc["R2"] == oc["R2"]
    assert qc["n_pairs"] == oc["n_valid_pairs"] and qc["n_valid"] == oc["n_valid_samples"]
    # perspective coordinates + broadcast ray dirs (point_query.py:95-108)
    from oracle import shade_oracle
    ref_loc = shade_oracle.w2pers(torch.from_numpy(o["sample_loc_w"]), torch.eye(3), torch.tensor(cfg.campos)).numpy()
    assert np.abs(loc - ref_loc).max() <= 1e-6
    assert np.array_equal(dirs[:, 0], rays["raydir"][0].numpy()[mask > 0])
    assert out[5] is opt.vsize


@pytest.mark.parametrize("name", ["tiny_opaque", "tiny_thin_sr8"])
def test_query_matches_reference_fixture(name, golden_dir):
    fx = golden.load(golden_dir, name)
    cfg = scene.CONFIGS["tiny"]
    net, pts, opt = harness.build_model(cfg, DEV, SR=int(fx["SR"]), max_o=100000)
    out = _query_points(net, scene.make_rays(cfg, fx["pixels"]))
    assert np.array_equal(out[4][0].cpu().numpy(), fx["ray_mask"])
    assert np.array_equal(out[0][0].cpu().numpy(), fx["sample_pidx"])
    assert np.array_equal(out[2][0].cpu().numpy(), fx["sample_loc_w"])
    assert np.abs(out[1][0].cpu().numpy() - fx["sample_loc"]).max() <= 1e-6
    assert np.array_equal(out[6], fx["ranges6"])


def test_query_train_jitter_table():
    """is_train: per-ray t table (jitter 0.3, point_query.py:81); same explicit table to both sides."""
    cfg = scene.CONFIGS["tiny"]
    net, pts, opt = harness.build_model(cfg, DEV)
    rays = scene.make_rays(cfg, scene.centre_patch(cfg, 30))
    R = rays["raydir"].shape[1]
    g = torch.Generator(device=DEV).manual_seed(7)
    t = device_t_table_jitter(cfg.near, cfg.far, cfg.D, R, 0.3, torch.device(DEV), generator=g)
    q = net.neural_points.querier.run_query(net.neural_points.xyz.detach(), rays["raydir"][0].to(DEV).contiguous(),
                                            list(cfg.campos), cfg.near, cfg.far, t=t, want_counters=True)
    from pointnerf_b200.point_query import make_cam_opts
    ex = q.export(make_cam_opts(cfg.campos, torch.eye(3)))
    o = _oracle(cfg, opt, pts, rays["raydir"][0], t=t.cpu().numpy())
    assert np.array_equal(ex["ray_mask"].cpu().numpy(), o["ray_mask"])
    assert np.array_equal(ex["sample_pidx"].cpu().numpy(), o["sample_pidx"])
    assert np.array_equal(ex["sample_loc_w"].cpu().numpy(), o["sample_loc_w"])


def test_query_edge_cases():
    cfg = scene.CONFIGS["tiny"]
    net, pts, opt = harness.build_model(cfg, DEV)
    rays = scene.make_rays(cfg, scene.centre_patch(cfg, 9))
    away = dict(rays); away["raydir"] = -rays["raydir"]
    out = _query_points(net, away)                       # nothing hit: empty R'
    assert out[0].shape == (1, 0, opt.SR, opt.K) and out[4].sum().item() == 0
    one = scene.make_rays(cfg, np.array([[cfg.W // 2, cfg.H // 2]], np.float32))
    out = _query_points(net, one)                        # a single ray
    o = _oracle(cfg, opt, pts, one["raydir"][0])
    _assert_same(out, o)
    # determinism: same call twice, bit-identical
    a = _query_points(net, rays); b = _query_points(net, rays)
    assert all(torch.equal(x, y) for x, y in zip(a[:5], b[:5]))
    # max_o overflow is reported through the counters, not resolved randomly
    net2, _, _ = harness.build_model(cfg, DEV, max_o=10)
    _query_points(net2, rays)
    assert net2.neural_points.querier.last_grid_counters["overflow_o"] == 1


def test_query_lego_scale_chunk_and_properties():
    """BASELINE config 2 size (N=400k, 258^3 voxels): one reference-sized chunk (2304 rays, run/train_ft.py:773)
    against the oracle, plus size-independent properties on the full 800x800 frame."""
    cfg = scene.CONFIGS["lego_render"]
    net, pts, opt = harness.build_model(cfg, DEV)
    chunk = scene.make_rays(cfg, scene.centre_patch(cfg, 48))
    out = _query_points(net, chunk)
    o = _oracle(cfg, opt, pts, chunk["raydir"][0])
    _assert_same(out, o)
    assert o["counters"]["overflow_o"] == 0 and o["counters"]["overflow_p"] == 0
    # full frame: sharding invariance -- every ray's result is independent of which rays share its call
    full = scene.make_rays(cfg)
    qr = net.neural_points.querier
    xyz = net.neural_points.xyz.detach()
    rd = full["raydir"][0].to(DEV).contiguous()
    q = qr.run_query(xyz, rd, list(cfg.campos), cfg.near, cfg.far, want_counters=True)
    cnt_full = dict(q.counters)
    from pointnerf_b200.point_query import make_cam_opts
    ex_full = q.export(make_cam_opts(cfg.campos, torch.eye(3)), want_pers=False, want_dirs=False)
    mask_full = ex_full["ray_mask"].clone(); pidx_full = ex_full["sample_pidx"].clone()
    R = rd.shape[0]
    tot = dict(n_cand=0, n_valid=0, n_pairs=0, R1=0, R2=0)
    rows = []
    for g in range(4):                                   # 4 interleaved shards (rank g takes rays g, g+4, ...)
        sel = torch.arange(g, R, 4, device=DEV)
        qs = qr.run_query(xyz, rd[sel].contiguous(), list(cfg.campos), cfg.near, cfg.far, want_counters=True)
        for k in tot:
            tot[k] += qs.counters[k]
        ex = qs.export(make_cam_opts(cfg.campos, torch.eye(3)), want_pers=False, want_dirs=False)
        assert torch.equal(ex["ray_mask"], mask_full[sel])
        rows.append((sel[ex["ray_mask"] > 0], ex["sample_pidx"].clone()))
    assert tot == {k: cnt_full[k] for k in tot}
    row_of = torch.cumsum((mask_full > 0).to(torch.int64), 0) - 1
    for sel_hit, pidx in rows:
        assert torch.equal(pidx_full[row_of[sel_hit]], pidx)
    assert 0.3 < cnt_full["R2"] / R < 0.6 and cnt_full["n_pairs"] <= cnt_full["n_valid"] * opt.K


@pytest.mark.parametrize("name,side", [("truck_8gpu", 40), ("scannet_8gpu", 32)])
def test_query_large_configs_chunk(name, side):
    """BASELINE configs 4/5 sizes (N=2M with kernel_size 5 / N=5M box with P=30): a reference-sized chunk vs oracle."""
    cfg = scene.CONFIGS[name]
    net, pts, opt = harness.build_model(cfg, DEV)
    rays = scene.make_rays(cfg, scene.centre_patch(cfg, side))
    out = _query_points(net, rays)
    o = _oracle(cfg, opt, pts, rays["raydir"][0])
    _assert_same(out, o)
    gc, oc = net.neural_points.querier.last_grid_counters, o["counters"]
    assert gc["n_occ"] == oc["n_occ"] and gc["max_pts"] == oc["max_pts"] and gc["overflow_p"] == oc["overflow_p"]
    assert o["counters"]["R2"] > 0
