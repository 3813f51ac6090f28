"""GPU: the probe outputs of point growing (opt.prob == 1, neural_points_volumetric_model.py:331-351) from k_probe_outputs
(pnb_probe_outputs), on the module's own query and opacity with an orbited camera (scene.orbit_rotation).

  bit for bit   the arg-max slot is torch.max(opacity, -1)'s (the first maximal slot); the opacity and position there are the
                composite's opacity and pnb_query_export's sample_loc_w at that slot; the weights are pnb_aux_outputs'
                weight * conf_coefficient at that slot; the full-R outputs (render_full(probe=True)) are the compacted ones on the hit
                rays and exact zeros elsewhere
  float64       ray_max_far_dist and the four averages against oracle/probe_oracle.py in float64 on the kernel's own export and
                opacity, as max |error| over max |value| of the key:
                  far_dist 4.5e-7, color 5e-7, dir 6.5e-7, conf 6e-7, embedding 4e-7
  whole frame   runner.probe_image equals probe_hole's 2304-ray chunk loop through forward() (runner.probe_image_chunked) bit for bit
                (is_train off); its coarse_raycolor and ray_mask equal runner.render_image's; a frame whose shading workspace
                overflowed is probed again and equals a clean run
Cases: K 1 / 3 / 8, SR 8 / 24 / 80, F 32 / 63, per-point frames; a transparent frame (alpha_bias -100: every opacity 0, the arg-max is
slot 0, whose K slots are all empty on many rays, so point 0 decides far_dist); a saturated one (alpha_bias 2000, raydist_mode_unit 0,
SR 80: opacities tie at 1.0 and the first slot must win; at alpha_bias 48 the tiny shell reaches 1.0 on one slot of a ray at most).
"""
import pytest
import torch

from oracle import probe_oracle
from pointnerf_b200 import harness, lib as L, runner, scene
from pointnerf_b200.point_query import make_cam_opts
from pointnerf_b200.ray_marching import _AuxFn, probe_keys, probe_outputs

pytestmark = pytest.mark.gpu
DEV = "cuda:0"
# 4-5x the largest error measured over CASES on an H100 80GB HBM3 (700 W): far_dist 9.7e-8, colour 1.04e-7, dir 1.44e-7, conf 1.25e-7,
# embedding 8.8e-8
BOUNDS = dict(ray_max_far_dist=4.5e-7, shading_avg_color=5e-7, shading_avg_dir=6.5e-7, shading_avg_conf=6e-7, shading_avg_embedding=4e-7)


def _build(K=8, SR=24, F=32, frames=False, alpha_bias=3.0, cfg_name="tiny", **over):
    cfg = scene.CONFIGS[cfg_name]
    net, pts, opt = harness.build_model(cfg, DEV, alpha_bias=alpha_bias, seed=2, feat_dim=F, K=K, SR=SR, prob=1, **over)
    if frames:
        net.neural_points.Rw2c = torch.nn.Parameter(scene.edit_frames(pts["xyz"]).to(DEV), requires_grad=False)
    return cfg, net


def _data(cfg, pixels=None, rotated=True):
    rays = scene.make_rays(cfg, pixels, camrotc2w=scene.orbit_rotation() if rotated else None)
    return {k: (v.to(DEV) if isinstance(v, torch.Tensor) else v) for k, v in rays.items()}


def _first_max(op):
    """First maximal slot of every row, written out (not through torch.max)."""
    SR = op.shape[-1]
    ar = torch.arange(SR, device=op.device).expand_as(op)
    return torch.where(op == op.max(-1, keepdim=True)[0], ar, torch.full_like(ar, SR)).min(-1)[0]


CASES = {
    "K8-SR24": dict(), "K1": dict(K=1), "K3-SR8": dict(K=3, SR=8), "SR80": dict(SR=80), "F63": dict(F=63), "frames": dict(frames=True),
    "K3-SR80-F63-frames": dict(K=3, SR=80, F=63, frames=True),
    "transparent": dict(alpha_bias=-100.0), "transparent-K3-F63": dict(alpha_bias=-100.0, K=3, F=63),
    "saturated": dict(alpha_bias=2000.0, SR=80, raydist_mode_unit=0),
}


@pytest.mark.parametrize("case", list(CASES))
def test_probe_outputs_bits_and_float64(case):
    over = CASES[case]
    cfg, net = _build(**over)
    data = _data(cfg)
    with torch.no_grad():
        full = net.render_full(data["campos"], data["raydir"], data["camrotc2w"], cfg.near, cfg.far, data["bg_color"], probe=True)
    net.check_errors()
    q = net.last
    q.counters = {k: int(v) for k, v in zip(L.QC, q.counters_tensor()[list(L.QC.values())].tolist())}   # for q.export (R')
    opacity = full["coarse_point_opacity"][0]
    mask = full["ray_mask"][0] > 0
    inds = torch.nonzero(mask)[:, 0]
    n = inds.shape[0]
    assert n > 0
    npn = net.neural_points
    F = int(npn.points_embeding.shape[-1])
    K = int(q.desc.K)
    with torch.no_grad():
        got = probe_outputs(net, q, opacity, inds, diag=True)
        wgt, cc, _ = _AuxFn.apply(net, q, inds, opacity, npn.points_conf)
    ex = q.export(make_cam_opts(list(q.desc.campos), data["camrotc2w"][0]), want_pers=False, want_dirs=False)
    op = opacity[inds]
    rows = torch.arange(n, device=DEV)
    slot = got["slot"].long()
    # bit for bit
    assert torch.equal(slot, torch.max(op, -1)[1]) and torch.equal(slot, _first_max(op))
    assert torch.equal(got["ray_max_shading_opacity"][:, 0], op[rows, slot])
    assert torch.equal(got["ray_max_sample_loc_w"], ex["sample_loc_w"][rows, slot])
    assert torch.equal(got["weight"], (wgt * cc)[rows, slot])
    for k, c in probe_keys(F):
        f = full[k][0]
        assert f.shape == (q.R, c) and got[k].shape == (n, c), k
        assert torch.equal(f[inds], got[k]), k
        assert torch.all(f[~mask] == 0), k
    # float64
    pts64 = dict(xyz=npn.xyz.detach().double(), embedding=npn.points_embeding.detach().double(), color=npn.points_color.detach().double(),
                 dir=npn.points_dir.detach().double(), conf=npn.points_conf.detach().double())
    ref = probe_oracle.probe(pts64, ex["sample_pidx"], ex["sample_loc_w"], op, dtype=torch.float64)
    assert torch.equal(ref["slot"], slot)
    errs = {k: float((got[k].double() - ref[k]).abs().max() / ref[k].abs().max().clamp(min=1e-30)) for k in BOUNDS}
    pidx = ex["sample_pidx"][rows, slot]
    empty = (pidx < 0).any(-1)
    d0 = (npn.xyz.detach()[0][None] - got["ray_max_sample_loc_w"]).norm(dim=-1)
    point0 = empty & (pidx < 0).all(-1)
    ties = int(((op == op.max(-1, keepdim=True)[0]).sum(-1) > 1).sum())
    print("\n[probe] %s: R'=%d, ties %d (slot>0 %d), max opacity %.4f, empty K slots at oi %d, all empty %d; errors %s"
          % (case, n, ties, int((slot > 0).sum()), float(op.max()), int(empty.sum()), int(point0.sum()),
             " ".join("%s %.2e" % (k.split("_")[-1], v) for k, v in errs.items())))
    for k, b in BOUNDS.items():
        assert errs[k] <= b, (k, errs[k])
    if 1 < K < 8 or over.get("alpha_bias", 0) < 0:
        assert int(empty.sum()) > 0                         # point 0 enters far_dist through empty slots
    if over.get("alpha_bias", 0) < 0:
        assert float(op.abs().max()) == 0.0 and torch.all(slot == 0)
        # on rays whose arg-max slot has no neighbour at all, far_dist is the distance to point 0
        assert int(point0.sum()) > 0
        assert torch.allclose(got["ray_max_far_dist"][point0, 0], d0[point0], rtol=1e-6, atol=0)
    if over.get("alpha_bias", 0) > 40:
        sat = (op == 1.0).sum(-1) > 1
        assert int(sat.sum()) > 0, "no ray has two saturated slots"
        assert torch.all(slot[sat] == _first_max(op[sat]))


@pytest.mark.parametrize("case", ["K8-SR24", "F63", "K3-SR80-F63-frames", "transparent"])
def test_probe_image_matches_chunk_loop(case):
    cfg, net = _build(**CASES[case])
    data = _data(cfg)
    maps = runner.probe_image(net, data, cfg.H, cfg.W)
    img = runner.render_image(net, data, cfg.H, cfg.W)
    chunked = runner.probe_image_chunked(net, data, cfg.H, cfg.W, 2304)
    net.check_errors()
    assert list(maps) == list(runner.PROBE_MAP_KEYS) and sorted(chunked) == sorted(maps)
    for k in maps:
        assert maps[k].dtype == chunked[k].dtype and torch.equal(maps[k], chunked[k]), k
    assert torch.equal(maps["coarse_raycolor"], img["coarse_raycolor"])
    assert torch.equal(maps["ray_mask"][..., 0], img["ray_mask"])
    miss = maps["ray_mask"][..., 0] == 0
    assert 0 < int(miss.sum()) < cfg.H * cfg.W
    for k in runner.PROBE_MAP_KEYS[2:]:
        assert torch.all(maps[k][miss] == 0), k


def test_probe_image_overflow_is_probed_again():
    """A frame denser than the shading workspace heuristic (the indoor scene: every ray keeps several valid samples, more than the 2
    per ray allowed here): probe_image sees the overflow, probes the frame again and returns what a module without the limit does."""
    cfg, small = _build(alpha_bias=3.0, K=8, SR=24, cfg_name="scannet_8gpu", pnb_max_valid_per_ray=2)
    data = _data(cfg, rotated=False)
    got = runner.probe_image(small, data, cfg.H, cfg.W)
    n_valid = int(small.last.counters_tensor()[L.QC["n_valid"]].item())
    assert small._valid_per_ray * cfg.H * cfg.W >= n_valid > 2 * cfg.H * cfg.W     # the first render overflowed; the retry was sized
    del small
    _, clean = _build(alpha_bias=3.0, K=8, SR=24, cfg_name="scannet_8gpu")
    want = runner.probe_image(clean, data, cfg.H, cfg.W)
    for k in want:
        assert torch.equal(want[k], got[k]), k


def test_probe_refusals():
    cfg, net = _build()
    data = _data(cfg, scene.centre_patch(cfg, 8))
    with torch.no_grad():
        full = net.render_full(data["campos"], data["raydir"], data["camrotc2w"], cfg.near, cfg.far, data["bg_color"])
    q = net.last
    lib = L.load()
    pts = net.neural_points.points_desc()
    bufs = [torch.zeros(q.R * 64, device=DEV) for _ in range(7)]
    args = lambda n_rows: (L.C.byref(q.desc), L.C.byref(pts), None, n_rows, full["coarse_point_opacity"][0].data_ptr(),
                           *[b.data_ptr() for b in bufs], None, None, torch.cuda.current_stream().cuda_stream)
    assert lib.pnb_probe_outputs(*args(q.R)) == 0
    assert lib.pnb_probe_outputs(*args(q.R - 1)) == -1        # without a row list, every ray
    for field, value in (("K", 9), ("SR", 129)):
        d = L.Query.from_buffer_copy(q.desc)
        setattr(d, field, value)
        assert lib.pnb_probe_outputs(L.C.byref(d), *args(q.R)[1:]) == -4, field
    p2 = net.neural_points.points_desc()
    p2.feat_dim = 48
    assert lib.pnb_probe_outputs(L.C.byref(q.desc), L.C.byref(p2), *args(q.R)[2:]) == -4
    torch.cuda.synchronize()
