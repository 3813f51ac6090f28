"""GPU: the fused module on the perspective-frustum query (wcoord_query 0), the DTU scripts' configuration (F = 63, point modes 01,
NN 2, SR 40, raydist_mode_unit 1, uniform jitter) on scene.FRUSTUM_CONFIGS["dtu_surface"] with an opaque surface, in every precision
and backward mode.  The reference is the eager shading of oracle/shade_oracle_frustum.py, restated with its per-sample outputs, both
agg_intrp_order values and given LeakyReLU masks in tests/frustum_shade_f64.py (held to it and to oracle/shade_oracle.py bit for bit by
tests/test_oracle_frustum_fused.py), in float64 on the drop-in querier's tuple (pointnerf_b200.query_point_indices), which is what the
reference's eager shading receives from that querier.

  forward      ray_mask and R' bit for bit; radiance, opacity and bg_T within 1e-4; the (sigma, rgb) of every valid sample within
               the per-sample bounds of DESIGN.md §6 item 6; the output keys of the reference module
  jitter       with is_train and one seed, the fused forward draws the drop-in's jitter (the same sample_loc)
  gradients    the colour loss (plain background, or the model shell's bg_ray formula through coarse_is_background) plus the
               zero_one loss on conf_coefficient, against float64 autograd of the oracle with the backward's own LeakyReLU masks
               (as tests/test_gpu_grad_f64.py does: with 501 block1.0 inputs the BF16x3 recompute takes ~1e-5 of the masks on the
               other side of zero, some 50 per step here, each moving one unit's row by up to ~5e-3 of scale), every point within
               oracle/grad_check.RTOL with no outlier allowance, the MLP tensors within grad_check.FRUSTUM_MLP_RTOL, alpha_branch.0
               with agg_intrp_order 1 within grad_check.ALPHA1_RTOL of its scale and ALPHA1_SUM_RTOL of each entry's sum |terms|
  whole frame  runner.render_image / probe_image bit for bit the 2304-ray chunk loops through forward(), with and without bg_ray,
               one build of the view; the probe outputs against oracle/probe_oracle.py in float64 within DESIGN §6's probe bounds
  bg_ray       for both queries, forward(bg_ray=...) is forward(bg_color=0) bit for bit, and the reference's fill_invalid on it is
               render_full(bg_ray=...) bit for bit
Every bound is one of DESIGN.md §6 or oracle/grad_check.py.  The file prints the errors it
measures (pytest -s).
"""
import functools
import json
import os

import numpy as np
import pytest
import torch

import frustum_shade_f64
from oracle import grad_check, probe_oracle
from pointnerf_b200 import harness, runner, scene
from pointnerf_b200 import query_point_indices as qpi
from pointnerf_b200.ray_marching import NeuralPoints, NeuralPointsRayMarching, PointAggregator, probe_keys

pytestmark = pytest.mark.gpu
DEV = torch.device("cuda:0")
TOL = 1e-4
CHUNK = 2304
MODES = {"bf16x3": dict(pnb_precision="bf16x3"), "bf16x3-general": dict(pnb_precision="bf16x3", pnb_frozen=0),
         "fp32": dict(pnb_precision="fp32")}
# DESIGN.md §6 item 6: sigma relative to the case's largest |sigma|, rgb absolute
SAMPLE_BOUNDS = {"bf16x3": (1.8e-5, 6e-6), "bf16x3-general": (2e-5, 7e-6), "fp32": (3e-6, 6e-7)}
# DESIGN.md §6, probe outputs against float64 (tests/test_gpu_probe.py), relative to each output's largest value
PROBE_BOUNDS = dict(ray_max_far_dist=4.5e-7, shading_avg_color=5e-7, shading_avg_dir=6.5e-7, shading_avg_conf=6e-7,
                    shading_avg_embedding=4e-7)
ZERO_EPS = 1e-3
MLP_RTOL = grad_check.FRUSTUM_MLP_RTOL


@functools.lru_cache(None)
def _scene():
    cfg = scene.FRUSTUM_CONFIGS["dtu_surface"]
    s = scene.make_frustum_scene(cfg)
    return cfg, s, scene.make_frustum_points(cfg, s)


def _opt(order=2, is_train=False, **over):
    cfg, _, _ = _scene()
    fo = vars(scene.frustum_opt(cfg, is_train=is_train))
    opt = harness.make_opt(scene.CONFIGS["tiny"], feat_dim=63, agg_intrp_order=order, **fo)
    for k, v in over.items():
        setattr(opt, k, v)
    return opt


def _net(order=2, is_train=False, mode="bf16x3", seed=5, **over):
    """The fused module on the frustum scene: its 63-channel points as stored (the oracle's), an opaque surface (alpha bias 300: the
    depth voxels are 0.0068 long)."""
    _, _, pts = _scene()
    opt = _opt(order, is_train, **MODES[mode], **over)
    agg = PointAggregator(opt, seed=seed)
    with torch.no_grad():
        agg.alpha_branch[0].bias += 300.0
    agg = agg.to(DEV)
    npn = NeuralPoints(opt, DEV)
    npn.set_points(pts["xyz"].to(DEV), pts["embedding"].to(DEV), points_color=pts["color"].to(DEV), points_dir=pts["dir"].to(DEV),
                   points_conf=pts["conf"].to(DEV), parameter=True, as_stored=True)
    assert isinstance(npn.querier, qpi.lighting_fast_querier)
    return NeuralPointsRayMarching(aggregator=agg, neural_points=npn, opt=opt), opt


def _data(pixels, bg=(1.0, 1.0, 1.0)):
    """The input dict of a reference dataset item for these pixels (directions through the pixel centres)."""
    cfg, s, _ = _scene()
    pix = np.asarray(pixels).reshape(-1, 2)
    K = s["intrinsic"]
    d = np.stack([(pix[:, 0] + 0.5 - K[0, 2]) / K[0, 0], (pix[:, 1] + 0.5 - K[1, 2]) / K[1, 1], np.ones(len(pix))], -1) @ s["camrotc2w"].T
    d = d / np.linalg.norm(d, axis=-1, keepdims=True)
    return dict(campos=torch.from_numpy(s["campos"]).to(DEV)[None], camrotc2w=torch.from_numpy(s["camrotc2w"]).to(DEV)[None],
                raydir=torch.from_numpy(d.astype(np.float32)).to(DEV)[None], pixel_idx=torch.from_numpy(pix.astype(np.int32)).to(DEV)[None],
                h=cfg.H, w=cfg.W, intrinsic=s["intrinsic"], near=cfg.near, far=cfg.far,
                bg_color=torch.tensor(bg, dtype=torch.float32, device=DEV))


def _forward(net, d, **kw):
    bg = kw.pop("bg_color", d["bg_color"])
    return net(d["campos"], d["raydir"], bg_color=bg, camrotc2w=d["camrotc2w"], pixel_idx=d["pixel_idx"], near=d["near"],
               far=d["far"], h=d["h"], w=d["w"], intrinsic=d["intrinsic"], **kw)


def _dropin(net, opt, d):
    """The drop-in querier's 7-tuple for the same view, as the reference's NeuralPoints obtains it (points in perspective coordinates
    by the reference's w2pers)."""
    cfg, _, _ = _scene()
    q = qpi.lighting_fast_querier(DEV, opt)
    xyz = net.neural_points.xyz.detach()
    pers = qpi.w2pers(xyz, d["camrotc2w"], d["campos"])
    return q.query_points(d["pixel_idx"], pers, xyz[None], torch.tensor([xyz.shape[0]], dtype=torch.int32), np.int64(cfg.H),
                          np.int64(cfg.W), d["intrinsic"], np.float32(cfg.near), np.float32(cfg.far), None, d["campos"],
                          d["camrotc2w"])


def _points_cpu(net, grad=False):
    npn = net.neural_points
    pts = dict(xyz=npn.xyz.detach().cpu(), embedding=npn.points_embeding.detach().cpu(), color=npn.points_color.detach().cpu(),
               dir=npn.points_dir.detach().cpu(), conf=npn.points_conf.detach().cpu(), Rw2c=torch.eye(3))
    if grad:
        for k in ("embedding", "color", "dir", "conf"):
            pts[k].requires_grad_(True)
    return pts


def _shade64(net, tup, d, order, bg, pts=None, mlp=None, slopes=None):
    pidx, loc, loc_w, dirs, _, vsize, _ = tup
    return frustum_shade_f64.shade(_points_cpu(net) if pts is None else pts, harness.mlp_cpu(net.aggregator) if mlp is None else mlp,
                                   pidx[0].cpu(), loc[0].detach().cpu(), loc_w[0].detach().cpu(), dirs[0].detach().cpu(),
                                   d["campos"].cpu(), d["camrotc2w"].cpu(), vsize, torch.as_tensor(bg, dtype=torch.float32).cpu(),
                                   dtype=torch.float64, agg_intrp_order=order, slopes=slopes)


def _check_forward(net, out, q, tup, ref, bounds, what):
    """Check 1 on one forward: mask and R' bit for bit, the 1e-4 rule, the per-sample bounds."""
    assert torch.equal(out["ray_mask"], tup[4]), what
    R2 = int(tup[0].shape[1])
    assert q.R2 == R2 and out["coarse_raycolor"].shape == (1, R2, 3), what
    errs = {}
    for k, rk in (("coarse_raycolor", "ray_color"), ("coarse_point_opacity", "opacity"), ("coarse_is_background", "bg_T")):
        errs[k] = float((out[k][0].detach().double().cpu().reshape(ref[rk].shape) - ref[rk]).abs().max())
    SR = q.SR
    sr = net._sigma_rgb[:R2 * SR].detach().double().cpu().view(R2, SR, 4)
    dec = ref["decoded"]
    valid = (tup[0][0] >= 0).any(-1).cpu()
    errs["sigma"] = float((sr[..., 0] - dec[..., 0])[valid].abs().max() / dec[..., 0][valid].abs().max())
    errs["rgb"] = float((sr[..., 1:] - dec[..., 1:])[valid].abs().max())
    print("\n[frustum fused] %s: R'=%d, valid samples %d, max opacity %.3f, errors %s"
          % (what, R2, int(valid.sum()), float(ref["opacity"].max()), " ".join("%s %.2e" % kv for kv in errs.items())))
    assert float(ref["opacity"].max()) > 0.5 and int(valid.sum()) > 1000        # an opaque surface, not all background
    for k in ("coarse_raycolor", "coarse_point_opacity", "coarse_is_background"):
        assert errs[k] <= TOL, (what, k, errs[k])
    assert errs["sigma"] <= bounds[0] and errs["rgb"] <= bounds[1], (what, errs)


def _pix_forward():
    _, s, _ = _scene()
    return s["pixel_idx"][::16]          # 1,200 rays: the float64 shading stays within a few GB


@functools.lru_cache(None)
def _forward_ref(order):
    net, opt = _net(order=order)
    d = _data(_pix_forward())
    tup = _dropin(net, opt, d)
    return tup, _shade64(net, tup, d, order, (1.0, 1.0, 1.0))


@pytest.mark.parametrize("order", [2, 1])
@pytest.mark.parametrize("mode", list(MODES))
def test_forward_matches_float64_oracle(golden_dir, mode, order):
    net, opt = _net(order=order, mode=mode)
    d = _data(_pix_forward())
    with torch.no_grad():
        out = _forward(net, d)
    q = net.last
    tup, ref = _forward_ref(order)
    _check_forward(net, out, q, tup, ref, SAMPLE_BOUNDS[mode], "%s order %d" % (mode, order))
    want = json.load(open(os.path.join(golden_dir, "output_keys.json")))["eval"]
    assert sorted(out) == sorted(want)
    assert out["conf_coefficient"].shape == (1, q.R2, opt.SR, opt.K) and out["queried_shading"].shape == (1, q.R2, 3)
    # queried_shading: 1 for a hit ray (its column is occupied) without any neighbour, as the reference's
    qs = (~(tup[0][0] >= 0).any(-1).any(-1)).float()
    assert torch.equal(out["queried_shading"][0, :, 0], qs)
    net.check_errors()


def test_jitter_is_the_drop_ins():
    """is_train with uniform jitter: the fused forward draws torch.rand([1, R', SR]) as the reference does, so one seed gives the
    drop-in's sample_loc; the radiance on that jitter meets check 1 (training runs the general pair kernel)."""
    net, opt = _net(is_train=True)
    d = _data(_pix_forward())
    torch.manual_seed(123)
    out = _forward(net, d)
    q = net.last
    torch.manual_seed(123)
    tup = _dropin(net, opt, d)
    assert torch.equal(q.sample_loc[None], tup[1])
    assert not torch.equal(tup[1][..., 2], _forward_ref(2)[0][1][..., 2])      # the jitter moved the samples
    ref = _shade64(net, tup, d, 2, (1.0, 1.0, 1.0))
    _check_forward(net, out, q, tup, ref, SAMPLE_BOUNDS["bf16x3-general"], "train jitter")
    net.check_errors()


# ------------------------------------------------------------------------------------------------ gradients
def _zero_one(cc):
    """The zero_one loss on conf_coefficient (models/base_rendering_model.py:629-641)."""
    val = torch.clamp(cc, ZERO_EPS, 1 - ZERO_EPS)
    return torch.mean(torch.log(val) + torch.log(1 - val))


def _pix_grad():
    _, s, _ = _scene()
    return s["pixel_idx"][::61]


def _bg_ray(n, seed=11):
    return torch.rand((1, n, 3), generator=torch.Generator().manual_seed(seed)).to(DEV)


def _grad_ref(net, tup, d, order, loss, slopes):
    """float64 autograd of the oracle on the drop-in's tuple, with the kernel's masks: the same loss, the gradients of every point
    group and MLP tensor."""
    pts = _points_cpu(net, grad=True)
    mlp = {k: v.detach().cpu().clone().requires_grad_(True) for k, v in net.aggregator.state_dict().items()}
    bg = (1.0, 1.0, 1.0) if loss == "color" else (0.0, 0.0, 0.0)
    with frustum_shade_f64.recording_softplus() as rec:
        r = _shade64(net, tup, d, order, bg, pts=pts, mlp=mlp, slopes=slopes)
    gt = _gt(int(tup[0].shape[1])).double()
    col = r["ray_color"]
    if loss == "bg_ray":
        hit = torch.nonzero(tup[4][0])[:, 0].cpu()
        col = r["bg_T"] * _bg_ray(d["pixel_idx"].shape[1])[0].cpu().double()[hit] + col
    pidx = tup[0][0].cpu()
    c0 = pts["conf"][0].double()[torch.clamp(pidx, min=0).long()][..., 0]          # neural_points.py:706-717
    cc = c0 - (c0 - torch.clamp(c0, min=0.0001, max=1)).detach()                     # point_aggregators.py:722-724
    L = ((col - gt) ** 2).sum() + 1e-3 * _zero_one(cc)
    L.backward()
    return dict(emb=pts["embedding"].grad, color=pts["color"].grad, dir=pts["dir"].grad, conf=pts["conf"].grad,
                mlp={k: v.grad for k, v in mlp.items()},
                abs_terms=frustum_shade_f64.alpha_branch_abs_terms(rec, r["hbar"]) if order == 1 else {})


def _gt(n):
    return torch.rand((n, 3), generator=torch.Generator().manual_seed(3))


@pytest.mark.parametrize("loss", ["color", "bg_ray"])
@pytest.mark.parametrize("order", [2, 1])
@pytest.mark.parametrize("precision,bwd_fp32", [("bf16x3", 0), ("bf16x3", 1), ("bf16x3", 4), ("fp32", 0), ("fp32", 1)])
def test_gradients_match_float64_autograd(precision, bwd_fp32, order, loss):
    mode = "bf16x3" if precision == "bf16x3" else "fp32"
    net, opt = _net(order=order, mode=mode, pnb_bwd_fp32=bwd_fp32)
    d = _data(_pix_grad())
    if loss == "color":
        out = _forward(net, d)
        col = out["coarse_raycolor"][0]
    else:
        bg_ray = _bg_ray(d["pixel_idx"].shape[1])
        out = _forward(net, d, bg_ray=bg_ray)
        hit = torch.nonzero(out["ray_mask"][0])[:, 0]
        col = out["coarse_is_background"][0] * bg_ray[0][hit] + out["coarse_raycolor"][0]     # the model shell's fill_invalid
    L = ((col - _gt(col.shape[0]).to(DEV)) ** 2).sum() + 1e-3 * _zero_one(out["conf_coefficient"][0])
    L.backward()
    tup = _dropin(net, opt, d)
    ref = _grad_ref(net, tup, d, order, loss, frustum_shade_f64.kernel_slopes(net, net.last))
    npn = net.neural_points
    rt = grad_check.RTOL[(bwd_fp32, precision)]
    got = dict(emb=npn.points_embeding.grad.cpu(), color=npn.points_color.grad.cpu(), dir=npn.points_dir.grad.cpu())
    errs = {k: float(grad_check.rel_point_errors(got[k], ref[k]).max()) for k in got}
    params = dict(net.aggregator.named_parameters())
    mlp = {k: grad_check.rel_error(p.grad.cpu(), ref["mlp"][k]) for k, p in params.items()}
    alpha1 = {k: (mlp[k], grad_check.sum_error(params[k].grad.cpu(), ref["mlp"][k], t), float(t.max() / ref["mlp"][k].abs().max()))
              for k, t in ref["abs_terms"].items()}
    worst = max((v, k) for k, v in mlp.items() if k not in alpha1)
    print("\n[frustum fused grads] %s/%d order %d %s: points %s | MLP worst %s %.2e%s" % (
        precision, bwd_fp32, order, loss, " ".join("%s %.2e" % kv for kv in errs.items()), worst[1], worst[0],
        "".join(" | %s %.2e of scale, %.2e of sum|terms| (sum|terms| %.0fx max|grad|)" % ((k,) + v) for k, v in alpha1.items())))
    for k in got:
        grad_check.check_points(got[k], ref[k], "points_" + k, rt[0])
    grad_check.check_conf(npn.points_conf.grad.cpu(), ref["conf"], int((tup[0] <= 0).sum()), rt[0])
    for k, e in mlp.items():
        if k in alpha1:
            continue
        assert e <= MLP_RTOL[(bwd_fp32, precision)], "aggregator.%s: %.3e of scale > %.1e" % (k, e, MLP_RTOL[(bwd_fp32, precision)])
    for k, (e, es, _) in alpha1.items():
        b, bs = grad_check.ALPHA1_RTOL[precision], grad_check.ALPHA1_SUM_RTOL[(bwd_fp32, precision)]
        assert e <= b, "aggregator.%s: %.3e of scale > %.1e" % (k, e, b)
        assert es <= bs, "aggregator.%s: %.3e of sum |terms| > %.1e" % (k, es, bs)
    assert npn.xyz.grad is None
    net.check_errors()


# ------------------------------------------------------------------------------------------------ whole frame
def _frame():
    _, s, _ = _scene()
    return s["pixel_idx"]


def test_render_image_is_the_chunk_loop():
    """runner.render_image (one call, fill_invalid in the kernel) equals the reference's 2304-ray chunk loop through forward() bit for
    bit, with the background colour and with bg_ray; every call of both reuses the one build of the view."""
    cfg, _, _ = _scene()
    net, opt = _net()
    d = _data(_frame())
    whole = runner.render_image(net, d, cfg.H, cfg.W)
    chunked = runner.render_image_chunked(net, d, cfg.H, cfg.W, CHUNK)
    assert np.array_equal(whole["coarse_raycolor"].cpu().numpy(), chunked["coarse_raycolor"])
    miss = whole["ray_mask"] == 0
    assert 0 < int(miss.sum()) < cfg.H * cfg.W
    bg_ray = _bg_ray(cfg.H * cfg.W)
    whole_b = runner.render_image(net, d, cfg.H, cfg.W, bg_ray=bg_ray)
    chunked_b = runner.render_image_chunked(net, d, cfg.H, cfg.W, CHUNK, bg_ray=bg_ray)
    assert np.array_equal(whole_b["coarse_raycolor"].cpu().numpy(), chunked_b["coarse_raycolor"])
    assert torch.equal(whole_b["coarse_raycolor"][miss], bg_ray[0].view(cfg.H, cfg.W, 3)[miss])
    assert not torch.equal(whole_b["coarse_raycolor"], whole["coarse_raycolor"])
    assert net.neural_points.querier.n_builds == 1
    net.check_errors()


def test_probe_image_is_the_chunk_loop_and_meets_the_probe_oracle():
    cfg, _, _ = _scene()
    net, opt = _net(prob=1)
    d = _data(_frame())
    maps = runner.probe_image(net, d, cfg.H, cfg.W)
    chunked = runner.probe_image_chunked(net, d, cfg.H, cfg.W, CHUNK)
    assert list(maps) == list(runner.PROBE_MAP_KEYS) and sorted(chunked) == sorted(maps)
    for k in maps:
        assert maps[k].dtype == chunked[k].dtype and torch.equal(maps[k], chunked[k]), k
    assert net.neural_points.querier.n_builds == 1
    # float64: the probe oracle on the drop-in's export and the fused opacity
    with torch.no_grad():
        full = net.render_full(d["campos"], d["raydir"], d["camrotc2w"], cfg.near, cfg.far, d["bg_color"], probe=True,
                               view={k: d[k] for k in ("pixel_idx", "h", "w", "intrinsic")})
    net.check_errors()
    tup = _dropin(net, opt, d)
    mask = full["ray_mask"][0] > 0
    assert torch.equal(full["ray_mask"], tup[4])
    inds = torch.nonzero(mask)[:, 0]
    op = full["coarse_point_opacity"][0][inds]
    npn = net.neural_points
    pts64 = dict(xyz=npn.xyz.detach().double(), embedding=npn.points_embeding.detach().double(), color=npn.points_color.detach().double(),
                 dir=npn.points_dir.detach().double(), conf=npn.points_conf.detach().double())
    ref = probe_oracle.probe(pts64, tup[0][0], tup[2][0], op, dtype=torch.float64)
    slot = torch.max(op, -1)[1]
    assert torch.equal(ref["slot"], slot)
    rows = torch.arange(inds.shape[0], device=DEV)
    assert torch.equal(full["ray_max_sample_loc_w"][0][inds], tup[2][0][rows, slot])
    errs = {k: float((full[k][0][inds].double() - ref[k]).abs().max() / ref[k].abs().max().clamp(min=1e-30)) for k in PROBE_BOUNDS}
    print("\n[frustum fused probe] R'=%d errors %s" % (inds.shape[0], " ".join("%s %.2e" % kv for kv in errs.items())))
    for k, b in PROBE_BOUNDS.items():
        assert errs[k] <= b, (k, errs[k])
    for k, c in probe_keys(63):
        assert torch.all(full[k][0][~mask] == 0), k


# ------------------------------------------------------------------------------------------------ bg_ray, both queries
def _reference_fill_bg_ray(out, bg_ray):
    """models/neural_points_volumetric_model.py:87-103 (fill_invalid with bg_ray) on a forward()'s outputs."""
    ray_mask = out["ray_mask"]
    B, OR = ray_mask.shape
    ray_inds = torch.nonzero(ray_mask)
    cib = torch.ones([B, OR, 1], dtype=out["coarse_is_background"].dtype, device=ray_mask.device)
    cib[ray_inds[..., 0], ray_inds[..., 1], :] = out["coarse_is_background"]
    col = cib * bg_ray
    col[ray_inds[..., 0], ray_inds[..., 1], :] += out["coarse_raycolor"][0]
    return col


def _world_net_and_data():
    cfg = scene.CONFIGS["tiny"]
    net, _, _ = harness.build_model(cfg, DEV, alpha_bias=3.0, feat_dim=63)
    rays = scene.make_rays(cfg, scene.centre_patch(cfg, 48))
    return net, {k: v.to(DEV) for k, v in rays.items()}, dict(near=cfg.near, far=cfg.far)


@pytest.mark.parametrize("query", ["world", "frustum"])
def test_bg_ray_is_no_background_then_fill_invalid(query):
    if query == "world":
        net, d, nf = _world_net_and_data()
        view = None
        run = lambda **kw: net(d["campos"], d["raydir"], camrotc2w=d["camrotc2w"], pixel_idx=d["pixel_idx"], near=d["near"],   # noqa: E731
                               far=d["far"], h=d["h"], w=d["w"], intrinsic=d["intrinsic"], **kw)
    else:
        net, _ = _net()
        d = _data(_pix_forward())
        nf = dict(near=d["near"], far=d["far"])
        view = {k: d[k] for k in ("pixel_idx", "h", "w", "intrinsic")}
        run = lambda **kw: _forward(net, d, **kw)                                                                # noqa: E731
    R = d["raydir"].shape[1]
    bg_ray = _bg_ray(R)
    with torch.no_grad():
        a = run(bg_color=torch.ones(3, device=DEV), bg_ray=bg_ray)
        b = run(bg_color=torch.zeros(3, device=DEV))
        full = net.render_full(d["campos"], d["raydir"], d["camrotc2w"], nf["near"], nf["far"], torch.ones(3), bg_ray=bg_ray, view=view)
    assert sorted(a) == sorted(b)
    for k in a:
        assert torch.equal(a[k], b[k]), k
    assert 0 < int(a["ray_mask"].sum()) < R
    assert torch.equal(full["coarse_raycolor"], _reference_fill_bg_ray(a, bg_ray))
    assert torch.equal(full["coarse_is_background"][0][a["ray_mask"][0] > 0], a["coarse_is_background"][0])
    net.check_errors()


# ------------------------------------------------------------------------------------------------ refusals, the reference module
def test_frustum_refusals():
    net, opt = _net()
    d = _data(_pix_forward()[:64])
    with pytest.raises(ValueError, match="pixel_idx"):
        net(d["campos"], d["raydir"], camrotc2w=d["camrotc2w"], near=d["near"], far=d["far"])
    npn = net.neural_points
    N = npn.xyz.shape[0]
    npn.Rw2c = torch.nn.Parameter(torch.eye(3, device=DEV).expand(N, 3, 3).contiguous(), requires_grad=False)
    with pytest.raises(NotImplementedError, match="per-point frames"):
        with torch.no_grad():
            _forward(net, d)
    for over in (dict(NN=1), dict(inverse=1)):
        with pytest.raises(NotImplementedError):
            qpi.lighting_fast_querier(DEV, _opt(**over))
    with pytest.raises(NotImplementedError, match="wcoord_query=0"):
        _net(point_features_dim=32)


def test_install_into_reference_shaped_module_with_the_frustum_querier():
    """Seam B (INTEGRATION.md) with a DTU-shaped module whose querier is the frustum drop-in: the native module's outputs."""
    import torch.nn as nn
    from pointnerf_b200 import ray_marching as P

    ours, opt = _net()
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
            self.querier = qpi.lighting_fast_querier(DEV, opt)

    class RefRayMarching(nn.Module):
        def __init__(self, aggregator, neural_points, opt):
            super().__init__()
            self.aggregator, self.neural_points, self.opt = aggregator, neural_points, opt

        def forward(self, *a, **k):
            raise AssertionError("the eager reference forward must have been replaced")

    P.install_into(RefRayMarching)
    net = RefRayMarching(ours.aggregator, RefNeuralPoints(), opt)
    d = _data(_pix_forward())
    with torch.no_grad():
        out = _forward(net, d)
        want = _forward(ours, d)
    assert sorted(out) == sorted(want)
    for k in want:
        assert torch.equal(out[k], want[k]), k
